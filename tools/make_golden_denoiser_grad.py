"""Generate tests/golden/denoiser_grad.npz with the REFERENCE's own Denoiser under torch autograd.

TEST INFRASTRUCTURE.  Run where the reference checkout (or the copy build() installs into oracle/_ref) is present:

    python tools/make_golden_denoiser_grad.py

`models.Denoiser` (models/denoiser.py:53-76) is imported unmodified through oracle/ref_loader.py (pytorch3d's HarmonicEmbedding
from oracle/shims) and run in fp32 on the CPU in eval mode (dropout off) with per-sample timesteps (0 and 99 in one batch) and
a random output gradient `ge` of eps.  Per case the file holds the inputs (z drawn fp16-representable and stored as float16),
eps, dL/dx, dL/dz and, with the scheme of oracle/make_golden_train.py, every parameter gradient of at most 512 elements in full
and a fingerprint (sum, L2 norm, 64 fixed samples) of every larger one; dL/dz is fingerprinted the same way.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader  # noqa: E402
from oracle.make_golden_train import sample_index  # noqa: E402
from posediffusion_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "denoiser_grad.npz")
STATE_SEED = 5
# name: (sequences, frames, seed)
CASES = {"b2n5": (2, 5, 1), "b3n20": (3, 20, 2), "b1n64": (1, 64, 3)}
FULL_MAX = 512  # gradients stored in full (larger ones are fingerprinted), so that the file stays a few hundred KB


def case_inputs(B, N, seed):
    """x [B,N,9], t [B] (0 and 99 included when B > 1), z [B,N,384], ge [B,N,9]."""
    g = torch.Generator().manual_seed(900 + seed)
    x = torch.randn(B, N, 9, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    t[0] = 0 if B > 1 else 42
    t[-1] = 99 if B > 1 else t[-1]
    z = torch.randn(B, N, 384, generator=g).half().float()  # fp16-representable: stored as float16, exactly
    ge = torch.randn(B, N, 9, generator=g)
    return x, t, z, ge


def fingerprint(a: np.ndarray) -> np.ndarray:
    flat = a.reshape(-1).astype(np.float64)
    return np.concatenate([[flat.sum(), np.linalg.norm(flat)], flat[sample_index(flat.size)]])


def main():
    ref = ref_loader.load_reference()
    torch.set_grad_enabled(True)
    state = syn.random_denoiser_state(STATE_SEED, 0.05)
    out = {"state_seed": np.array([STATE_SEED], dtype=np.int64)}
    for name, (B, N, seed) in CASES.items():
        den = ref.Denoiser(TRANSFORMER=ref.to_attr(ref_loader.TRANSFORMER_CFG))
        den.load_state_dict(state, strict=True)
        den.eval()  # dropout off
        x, t, z, ge = case_inputs(B, N, seed)
        xx, zz = x.clone().requires_grad_(True), z.clone().requires_grad_(True)
        eps = den(xx, t, zz)
        (eps * ge).sum().backward()
        p = f"{name}_"
        for k, v in (("x", x), ("t", t), ("ge", ge)):
            out[p + k] = v.numpy()
        out[p + "z"] = z.half().numpy()
        out[p + "eps"] = eps.detach().numpy()
        out[p + "dx"] = xx.grad.numpy()
        out[p + "fp:dz"] = fingerprint(zz.grad.numpy())
        for pname, prm in den.named_parameters():
            gr = prm.grad.detach().numpy().astype(np.float32)
            if gr.size <= FULL_MAX:
                out[f"{p}grad:{pname}"] = gr
            else:
                out[f"{p}fp:{pname}"] = fingerprint(gr)
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
