"""GPU test of pdb_cameras_align / posediffusion_b200.corresponding_cameras_alignment (demo.py:126-128).

Written in a session without GPU access.  What was verified without a GPU: the device maths on the host (same __host__ __device__
functions, tests/test_alignment_cpu.py), and the two kernel bodies on the CPU emulation of the execution model with the
entry point's launch geometry (tests/host/cuda_emu.h).  The file sorts last among the GPU tests on purpose: it is the one
test module whose kernels ran last on the GPU when it was written.
"""
import numpy as np
import pytest
import torch

from oracle import cameras_alignment as oca

import posediffusion_b200 as pdb
from posediffusion_b200 import metric
from test_alignment_cpu import as_t, similarity_scene

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n,noise,estimate_scale", [(1, 0.0, True), (2, 0.0, True), (5, 0.05, True), (20, 0.2, True), (20, 0.2, False), (80, 0.02, True)])
def test_cameras_align_matches_oracle(n, noise, estimate_scale):
    R_src, T_src, R_tgt, T_tgt, _ = similarity_scene(n, seed=100 + n, noise=noise)
    ts = as_t(R_src, T_src, R_tgt, T_tgt)
    src = pdb.PerspectiveCameras(focal_length=torch.ones(n, 2).cuda(), R=ts[0].cuda(), T=ts[1].cuda())
    tgt = pdb.PerspectiveCameras(focal_length=torch.ones(n, 2), R=ts[2], T=ts[3])  # host targets are moved to the device
    out = pdb.corresponding_cameras_alignment(src, tgt, estimate_scale=estimate_scale, mode="extrinsics", eps=1e-9)
    want_R, want_T = oca.corresponding_cameras_alignment(*ts, estimate_scale=estimate_scale)
    np.testing.assert_allclose(out.R.cpu().numpy(), want_R.numpy(), atol=1e-5)
    np.testing.assert_allclose(out.T.cpu().numpy(), want_T.numpy(), atol=3e-5 * max(1.0, want_T.abs().max().item()))
    assert out.focal_length is src.focal_length and len(out) == n


def test_similarity_is_undone_and_are_vanishes():
    """The demo's metric: after alignment the absolute rotation error of similarity-transformed cameras is ~0."""
    R_src, T_src, R_tgt, T_tgt, _ = similarity_scene(20, seed=7)
    ts = as_t(R_src, T_src, R_tgt, T_tgt)
    src = pdb.PerspectiveCameras(focal_length=torch.ones(20, 2).cuda(), R=ts[0].cuda(), T=ts[1].cuda())
    tgt = pdb.PerspectiveCameras(focal_length=torch.ones(20, 2).cuda(), R=ts[2].cuda(), T=ts[3].cuda())
    before = metric.compute_ARE(src.R, tgt.R).mean()
    aligned = pdb.corresponding_cameras_alignment(src, tgt)
    after = metric.compute_ARE(aligned.R, tgt.R).mean()
    assert before > 5.0 and after < 0.2  # acos near 1 turns one fp32 ulp of the trace into 0.02 degrees
    np.testing.assert_allclose(aligned.T.cpu().numpy(), T_tgt, atol=1e-4 * max(1.0, np.abs(T_tgt).max()))
