"""Host-side pieces of the backbone training path: workspace sizing, the new ABI symbols, and the float64 gradient oracle."""
import ctypes as C

import torch

from oracle import vit_train_oracle as vo
from oracle.dino_vit import DinoViTSmall16, multiscale_features, randomize
from posediffusion_b200 import _native

DEFAULT = (1, 1 / 2, 1 / 3)


def test_workspace_bytes_monotonic_zero_when_unsupported_and_within_budget():
    sizes = [_native.vit_train_workspace_bytes(n, 224, 224, DEFAULT) for n in (1, 2, 7, 21, 128, 512)]
    assert all(a > 0 for a in sizes) and all(a < b for a, b in zip(sizes, sizes[1:]))
    assert sizes[-1] < 40 * 2**30, sizes[-1]  # beside the denoiser's 8.4 GB on an 80 GB card
    assert _native.vit_train_workspace_bytes(2, 224, 232, DEFAULT) > 0
    for bad in ((0, 224, 224, DEFAULT), (1, 224, 224, ()), (1, 224, 224, (1, 1, 1, 1, 1)), (1, 8, 8, DEFAULT), (1, 512, 512, (1,)),
                (1, 224, 224, (1, -0.5)), (70000, 224, 224, DEFAULT)):
        assert _native.vit_train_workspace_bytes(*bad) == 0, bad


def test_new_symbols_are_additions_to_abi_version_2():
    lib = _native.load_library()
    assert lib.pdb_abi_version() == 2
    for name in ("pdb_train_backward_z", "pdb_vit_train_workspace_bytes", "pdb_vit_train_forward", "pdb_vit_backward"):
        assert hasattr(lib, name)
    assert lib.pdb_vit_train_forward(None, None, None, 1, 224, 224, None, 1, None, None, None) == _native.PDB_ERR_INVALID
    assert lib.pdb_vit_backward(None, None, None, None, None, None) == _native.PDB_ERR_INVALID
    assert lib.pdb_train_backward_z(None, None, None, None, None, None, None, None) == _native.PDB_ERR_INVALID


def test_oracle_matches_fp32_autograd_of_the_restated_network():
    """The float64 oracle against plain fp32 autograd through oracle/dino_vit.py (non-square input: resampled position grid)."""
    vit = randomize(DinoViTSmall16(), 11)
    img = torch.rand(1, 3, 224, 232, generator=torch.Generator().manual_seed(1))
    g = torch.randn(1, 384, generator=torch.Generator().manual_seed(2))
    z = multiscale_features(vit, img, DEFAULT)
    (z * g).sum().backward()
    zr, ref = vo.features_and_grads(vit.state_dict(), img, DEFAULT, g)
    assert (z.detach().double() - zr).abs().max().item() < 1e-4
    for name, p in vit.named_parameters():
        d = ((p.grad.double() - ref[name]).norm() / ref[name].norm()).item()
        assert d < 1e-4, (name, d)
    _, tf = vo.features_and_grads(vit.state_dict(), img, DEFAULT, g, tf32=True)
    d = max(((tf[k] - ref[k]).norm() / ref[k].norm()).item() for k in ref)
    assert 1e-6 < d < 5e-2, d  # the TF32 run is a different, nearby computation
