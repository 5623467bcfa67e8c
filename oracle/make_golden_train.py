"""Generate tests/golden/train.npz with the REFERENCE's own training step and camera encoding.

TEST INFRASTRUCTURE.  Run where the reference checkout (or the copy build() installs into oracle/_ref) is present:

    python -m oracle.make_golden_train

`models.GaussianDiffusion.p_losses` around `models.Denoiser` (models/gaussian_diffuser.py:308-341) are imported unmodified through
oracle/ref_loader.py and run in fp32 on the CPU with dropout off (eval mode), injected `t` and noise, and random output
gradients `gl` (of `loss`) and `gx` (of `x_0_pred`); the backward is torch autograd.  Per case the file holds the inputs, `x_t`,
`x_0_pred`, `loss`, the full gradients of every tensor with at most 2048 elements, and for every larger tensor a fingerprint:
sum, L2 norm and the values at 64 fixed flat indices (the full 17.3 M gradients do not belong in git).

`util/camera_transform.camera_to_pose_encoding` (:108-129) is run on rotations that take each of the four branches of
`matrix_to_quaternion` and on focal lengths beyond both clamp bounds.  pytorch3d is not installed; its `matrix_to_quaternion`
is supplied, for this run, by `oracle.train_oracle.matrix_to_quaternion` (the standardised form: real part >= 0), installed
into the pytorch3d shim module and into the reference module that imported the name.
"""
from __future__ import annotations

import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import ref_loader, train_oracle  # noqa: E402
from posediffusion_b200 import synthetic as syn  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "train.npz")
# name: (sequences, frames, batch_repeat, loss_type, seed)
CASES = {"b2n5": (2, 5, 1, "l1", 1), "b3n20": (3, 20, 1, "l2", 2), "repeat3": (2, 4, 3, "l1", 3)}
FULL_MAX = 2048
SAMPLES = 64


def sample_index(numel: int) -> np.ndarray:
    return (np.arange(SAMPLES, dtype=np.int64) * 7919 + 13) % numel


def case_inputs(seqs, frames, repeat, seed):
    """x_start [seqs*repeat, frames, 9], z [seqs, frames, 384] (repeated like PoseDiffusionModel), t, noise, gl, gx."""
    g = torch.Generator().manual_seed(500 + seed)
    B = seqs * repeat
    x = torch.randn(B, frames, 9, generator=g) * 0.5
    z = torch.randn(seqs, frames, 384, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    noise = torch.randn(B, frames, 9, generator=g)
    gl = torch.randn(B, frames, 9, generator=g)
    gx = torch.randn(B, frames, 9, generator=g)
    return x, z, t, noise, gl, gx


def camera_inputs():
    """Rotations (each matrix_to_quaternion branch) from quaternions, translations, focal lengths (some beyond both bounds)."""
    g = torch.Generator().manual_seed(77)
    q = torch.randn(32, 4, generator=g)
    q[:4] = torch.tensor([[1.0, 0.1, 0.05, 0.02], [0.05, 1.0, 0.1, 0.02], [0.02, 0.1, 1.0, 0.05], [0.05, 0.02, 0.1, 1.0]])
    q[4:8] *= -1.0  # negative real parts: the standardisation flips them
    from oracle.shims.pytorch3d.transforms.rotation_conversions import quaternion_to_matrix

    R = quaternion_to_matrix(q)
    T = torch.randn(32, 3, generator=g)
    focal = torch.exp(torch.randn(32, 2, generator=g) * 2.0)
    focal[0] = torch.tensor([0.01, 50.0])
    focal[1] = torch.tensor([0.1, 20.0])
    return R, T, focal


def main():
    ref = ref_loader.load_reference()
    from pytorch3d.transforms import rotation_conversions  # the shim, on sys.path after load_reference
    from util import camera_transform

    rotation_conversions.matrix_to_quaternion = train_oracle.matrix_to_quaternion
    camera_transform.matrix_to_quaternion = train_oracle.matrix_to_quaternion
    torch.set_grad_enabled(True)
    out = {}
    state = syn.random_denoiser_state(3, 0.05)
    out["state_seed"] = np.array([3], dtype=np.int64)
    for name, (seqs, frames, repeat, loss_type, seed) in CASES.items():
        den = ref.Denoiser(TRANSFORMER=ref.to_attr(ref_loader.TRANSFORMER_CFG))
        den.load_state_dict(state, strict=True)
        dif = ref.GaussianDiffusion(beta_schedule="custom", loss_type=loss_type)
        dif.model = den
        dif.eval()  # dropout off
        x, z, t, noise, gl, gx = case_inputs(seqs, frames, repeat, seed)
        res = dif.p_losses(x, t, z=z.repeat(repeat, 1, 1), noise=noise)
        total = (res["loss"] * gl).sum() + (res["x_0_pred"] * gx).sum()
        total.backward()
        p = f"{name}_"
        for k, v in (("x_start", x), ("z", z), ("t", t), ("noise", noise), ("gl", gl), ("gx", gx)):
            out[p + k] = v.numpy()
        for k in ("x_t", "x_0_pred", "loss"):
            out[p + k] = res[k].detach().numpy()
        for pname, prm in den.named_parameters():
            gr = prm.grad.detach().numpy().astype(np.float32)
            if gr.size <= FULL_MAX:
                out[f"{p}grad:{pname}"] = gr
            else:
                flat = gr.reshape(-1).astype(np.float64)
                out[f"{p}fp:{pname}"] = np.concatenate([[flat.sum(), np.linalg.norm(flat)], flat[sample_index(flat.size)]])
    R, T, focal = camera_inputs()
    cams = SimpleNamespace(R=R, T=T, focal_length=focal)
    out["cam_R"], out["cam_T"], out["cam_focal"] = R.numpy(), T.numpy(), focal.numpy()
    out["cam_pose"] = camera_transform.camera_to_pose_encoding(cams).numpy()
    np.savez_compressed(OUT, **out)
    print(f"wrote {OUT}: {len(out)} arrays, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
