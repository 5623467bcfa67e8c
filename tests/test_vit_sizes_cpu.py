"""CPU checks behind tests/test_gpu_vit_sizes.py: the position-table helper at every grid the attention kernel accepts, and the
float64 extractor oracle (oracle/vit_f64.py) pinned to the existing oracle and to the reference's fixtures."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle.dino_vit import DinoViTSmall16, multiscale_features, randomize
from oracle.make_golden_features import CASES, VIT_SEED, images_for
from oracle.train_oracle import _linear
from oracle.vit_f64 import VitF64
from posediffusion_b200 import _native


@pytest.fixture(scope="module")
def net():
    return randomize(DinoViTSmall16(), VIT_SEED).eval()


def test_position_table_helper_at_every_grid_up_to_255_patches():
    """pdb_vit_pos_table against float64 torch bicubic (the hub model's interpolate_pos_encoding) for every gh x gw <= 255;
    (14, 14) is the square input and returns the stored table bit for bit.  2e-5 on values up to 4.5: float32 evaluation
    (torch's own float32 bicubic is 9e-6 from float64 here); a wrong tap or coefficient is off by O(0.1)."""
    pos = torch.randn(1, 197, 384, generator=torch.Generator().manual_seed(7))
    side = pos[:, 1:].double().reshape(1, 14, 14, 384).permute(0, 3, 1, 2)
    grids = [(gh, gw) for gh in range(1, 256) for gw in range(1, 256 // gh + 1) if gh * gw <= 255]
    assert len(grids) > 1000
    for gh, gw in grids:
        out = _native.vit_pos_table(pos.numpy(), gh, gw)
        if (gh, gw) == (14, 14):
            assert np.array_equal(out, pos[0].numpy())
            continue
        grid = F.interpolate(side, scale_factor=((gh + 0.1) / 14, (gw + 0.1) / 14), mode="bicubic")
        assert tuple(grid.shape[-2:]) == (gh, gw)
        assert np.array_equal(out[0], pos[0, 0].numpy()), (gh, gw)
        err = np.abs(out[1:] - grid[0].permute(1, 2, 0).reshape(-1, 384).numpy()).max()
        assert err <= 2e-5, (gh, gw, err)


@pytest.mark.parametrize("case", list(CASES))
def test_f64_oracle_is_pinned_to_multiscale_features_and_the_fixtures(net, golden, case):
    """In float32 the evaluator is multiscale_features (1e-5); in float64 it is within twice the float32 run's distance of the
    reference's own fixture."""
    n, h, w, sf, seed = CASES[case]
    img = images_for(n, h, w, seed)
    with torch.no_grad():
        ref = multiscale_features(net, img, sf)
    z32 = VitF64(net.state_dict(), torch.float32).features(img, sf)
    assert (z32 - ref).abs().max().item() <= 1e-5
    z64 = VitF64(net.state_dict()).features(img, sf)
    d32 = (z32.double() - z64).abs().max().item()
    gold = torch.from_numpy(golden("features.npz")[case]).double()
    assert 0 < d32 < 1e-4
    assert (gold - z64).abs().max().item() <= 2 * d32, ((gold - z64).abs().max().item(), d32)


def test_folded_tf32_with_unit_affine_is_the_plain_tf32_matmul(net):
    """With gamma = 1 and beta = 0 the fold is the identity (W' = W, b' = b, colsum = row sums of W), so block k in "tf32" mode
    equals the block written with the training oracle's TF32 matmul and LayerNorm's centring applied after it."""
    state = {k: v.clone() for k, v in net.state_dict().items()}
    for k in state:
        if ".norm1." in k or ".norm2." in k:
            state[k] = torch.ones_like(state[k]) if k.endswith("weight") else torch.zeros_like(state[k])
    ev = VitF64(state)
    P = ev.p
    x = 3.0 + torch.randn(2, 50, 384, generator=torch.Generator().manual_seed(4), dtype=torch.float64)
    for k in (1, 7, 12):
        pre = f"blocks.{k - 1}."
        wf, colsum, bf = ev.folded[(k - 1, "qkv")]
        assert torch.equal(wf, P[pre + "attn.qkv.weight"]) and torch.equal(bf, P[pre + "attn.qkv.bias"])

        def ln_lin(v, name):
            w, b = P[pre + name + ".weight"], P[pre + name + ".bias"]
            mean = v.mean(-1, keepdim=True)
            rstd = ((v - mean).pow(2).mean(-1, keepdim=True) + 1e-6).rsqrt()
            return rstd * (_linear(v, w, torch.zeros_like(b), "trunc") - mean * w.sum(1)) + b

        y = x + _linear(ev.attention(ln_lin(x, "attn.qkv"), "tf32"), P[pre + "attn.proj.weight"], P[pre + "attn.proj.bias"], "trunc")
        want = y + _linear(F.gelu(ln_lin(y, "mlp.fc1")), P[pre + "mlp.fc2.weight"], P[pre + "mlp.fc2.bias"], "trunc")
        got = ev.block(k, x, "tf32")
        assert (got - want).abs().max().item() <= 1e-12 * want.abs().max().item(), k
        # and the rounding is real: the TF32 block is measurably, but only TF32-far, from float64
        d = (got - ev.block(k, x)).abs().max().item() / (want - x).abs().max().item()
        assert 1e-6 < d < 1e-2, (k, d)
