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


def test_chunked_oracle_equals_one_call():
    """features_and_grads_chunked (chunks of 2, 2 and 1 images, two scales) vs one features_and_grads call, both roundings."""
    state = randomize(DinoViTSmall16(), 5).state_dict()
    img = torch.rand(5, 3, 32, 48, generator=torch.Generator().manual_seed(3))
    g = torch.randn(5, 384, generator=torch.Generator().manual_seed(4))
    for tf32 in (False, True):
        z1, g1 = vo.features_and_grads(state, img, (1, 1 / 2), g, tf32=tf32)
        z2, g2 = vo.features_and_grads_chunked(state, img, (1, 1 / 2), g, tf32=tf32, chunk=2)
        assert ((z2 - z1).norm() / z1.norm()).item() <= 1e-12
        assert set(g1) == set(g2)
        for k in g1:
            assert ((g2[k] - g1[k]).norm() / g1[k].norm().clamp(min=1e-30)).item() <= 1e-12, k


def test_position_table_gradient_is_the_adjoint_of_the_resampling():
    """The oracle's and the restated network's position tables are F.interpolate's bicubic forward, and their d pos_embed is
    R_s^T applied to the table's gradient, with R_s read off the forward one stored cell at a time; 14x14 of a non-square image
    included (torch's own bicubic backward copies the gradient through at that size)."""
    import torch.nn.functional as F

    from oracle.vit_f64 import VitF64

    vit = randomize(DinoViTSmall16(), 5)
    state = vit.state_dict()
    for gh, gw in ((14, 14), (16, 7), (1, 31), (1, 1)):
        ev = VitF64(state)
        grid = ev.p["pos_embed"][0, 1:].reshape(1, 14, 14, -1).permute(0, 3, 1, 2)
        direct = F.interpolate(grid, scale_factor=((gh + 0.1) / 14, (gw + 0.1) / 14), mode="bicubic")[0].permute(1, 2, 0).reshape(gh * gw, -1)
        torch.testing.assert_close(ev.pos_table(gh, gw, 16 * gh, 16 * gw + 1)[1:], direct, rtol=0, atol=1e-12)
        with torch.no_grad():
            net = vit.interpolate_pos_encoding(gh * gw, 16 * gh, 16 * gw + 1)[0, 1:]
        torch.testing.assert_close(net.double(), direct, rtol=0, atol=1e-6)
        pos = ev.p["pos_embed"].clone().requires_grad_(True)
        ev.p["pos_embed"] = pos
        y = ev.pos_table(gh, gw, 16 * gh, 16 * gw + 1)
        g = torch.randn_like(y)
        (got,) = torch.autograd.grad((y * g).sum(), pos)
        # stored row k set to ones, the rest zero: the table is column k of the map in every channel, so summing
        # (table * g) gives sum over channels of (map^T g)[k]
        want = []
        with torch.no_grad():
            for k in range(197):
                ev.p["pos_embed"] = torch.zeros_like(pos)
                ev.p["pos_embed"][0, k] = 1.0
                want.append((ev.pos_table(gh, gw, 16 * gh, 16 * gw + 1) * g).sum())
        torch.testing.assert_close(got[0].sum(-1), torch.stack(want), rtol=0, atol=1e-9, msg=f"{gh}x{gw}")
