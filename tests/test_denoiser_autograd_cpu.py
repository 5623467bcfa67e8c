"""Differentiable Denoiser.forward without a GPU: the float64 oracle it is tested against (tests/denoiser_grad_oracle.py) against
oracle/train_oracle.py and torch's own modules, against the reference's fp32 fixture (tests/golden/denoiser_grad.npz), and the
Python refusals that need no device."""
import numpy as np
import pytest
import torch

import posediffusion_b200 as pdb
from denoiser_grad_oracle import denoiser_eps, eps_and_grads
from oracle import pose_oracle as po
from oracle import train_oracle as to
from oracle.make_golden_train import sample_index
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
GOLDEN_CASES = ("b1n64", "b2n5", "b3n20")


def test_denoiser_eps_equals_forward_eps_at_x_t():
    state = syn.random_denoiser_state(2, 0.05)
    params = {k: v.double() for k, v in state.items()}
    B, N = 3, 6
    g = torch.Generator().manual_seed(0)
    x, noise = torch.randn(B, N, 9, generator=g), torch.randn(B, N, 9, generator=g)
    t = torch.tensor([0, 57, 99])
    z = syn.random_features(B, N, 1)
    masks = to.dropout_masks(17, 0, B, N, 0.1)
    for m, p in ((None, 0.0), (masks, 0.1)):
        out = to.forward(params, x, t, noise, z, "l1", m, p)
        assert torch.equal(denoiser_eps(params, out["x_t"], t, z, m, p), out["eps"])
        out = to.forward(params, x, t, noise, z, "l1", m, p, tf32="trunc")
        assert torch.equal(denoiser_eps(params, out["x_t"], t, z, m, p, tf32="trunc"), out["eps"])


def test_gradients_match_torch_autograd_through_the_oracle_modules():
    """dx, dz and the parameter gradients against nn.TransformerEncoder in float64 (dropout 0) with the shim's harmonic
    embedding (the reference's pose_embed, differentiable in x)."""
    from oracle.shims.pytorch3d.renderer import HarmonicEmbedding

    state = syn.random_denoiser_state(4, 0.05)
    net = po.build_denoiser(state).double().train()
    for m in net.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
        if isinstance(m, torch.nn.MultiheadAttention):
            m.dropout = 0.0
    embed = HarmonicEmbedding(n_harmonic_functions=10).double()
    B, N = 2, 5
    g = torch.Generator().manual_seed(1)
    x = torch.randn(B, N, 9, generator=g, dtype=torch.float64, requires_grad=True)
    z = syn.random_features(B, N, 2).double().requires_grad_(True)
    t = torch.tensor([3, 80])
    ge = torch.randn(B, N, 9, generator=g, dtype=torch.float64)
    temb = net.time_embed.linear(po.timestep_features(t).double())[:, None, :].expand(-1, N, -1)
    pivot = torch.zeros(B, N, 1, dtype=torch.float64)
    pivot[:, 0] = 1.0
    eps = net._last(net._trunk(net._first(torch.cat([embed(x), temb, z, pivot], dim=-1))))
    (eps * ge).sum().backward()
    got_eps, grads, dx, dz = eps_and_grads(state, x, t, z, ge)
    torch.testing.assert_close(got_eps, eps.detach(), rtol=1e-9, atol=1e-12)
    torch.testing.assert_close(dx, x.grad, rtol=1e-9, atol=1e-12)
    torch.testing.assert_close(dz, z.grad, rtol=1e-9, atol=1e-12)
    named = dict(net.named_parameters())
    for n, gr in grads.items():
        torch.testing.assert_close(gr, named[n].grad, rtol=1e-9, atol=1e-12, msg=n)


def golden_inputs(g, name):
    T = lambda k: torch.from_numpy(g[f"{name}_{k}"].astype(np.float32) if k == "z" else g[f"{name}_{k}"])  # noqa: E731
    return T("x"), T("t"), T("z"), T("ge")


def golden_distance(g, name, eps, dx, dz, grads):
    """As tests/test_train_cpu.py's: relative L2 distance per tensor; a fingerprinted tensor n gives key n (norm and sum bound)
    and key (n, "samples") (64 samples)."""
    p = f"{name}_"
    rel = lambda a, b: float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-30))  # noqa: E731
    out = {"eps": rel(eps, g[p + "eps"]), "dx": rel(dx, g[p + "dx"])}
    for n, gr in {**grads, "dz": dz}.items():
        a = np.asarray(gr, np.float64)
        if p + "grad:" + n in g:
            out[n] = rel(a, g[p + "grad:" + n])
        else:
            fp, flat = g[p + "fp:" + n], a.reshape(-1)
            out[n] = max(abs(np.linalg.norm(flat) - fp[1]) / fp[1], abs(flat.sum() - fp[0]) / (fp[1] * np.sqrt(flat.size)))
            out[(n, "samples")] = rel(flat[sample_index(flat.size)], fp[2:])
    return out


def as_dict(eps, grads, dx, dz):
    return {"eps": eps, "dx": dx, "dz": dz, **grads}


def full_distance(a, b):
    return {k: float((a[k].double() - b[k].double()).norm() / b[k].double().norm().clamp(min=1e-30)) for k in b}


@pytest.mark.parametrize("name", GOLDEN_CASES)
def test_oracle_against_reference_goldens(golden, name):
    """Float64 oracle vs the reference's own fp32 Denoiser under autograd, with the bound tests/test_train_cpu.py uses for
    train.npz: twice the float32 oracle's distance from float64 plus 1e-6, four times that for a 64-sample estimate."""
    g = golden("denoiser_grad.npz")
    state = syn.random_denoiser_state(int(g["state_seed"][0]), 0.05)
    x, t, z, ge = golden_inputs(g, name)
    ref = eps_and_grads(state, x, t, z, ge)
    d32 = full_distance(as_dict(*eps_and_grads(state, x, t, z, ge, dtype=torch.float32)), as_dict(*ref))
    got = golden_distance(g, name, ref[0].numpy(), ref[2].numpy(), ref[3].numpy(), {n: v.numpy() for n, v in ref[1].items()})
    assert len(got) > 110
    for k, d in got.items():
        base = d32[k[0] if isinstance(k, tuple) else k]
        bound = (4 if isinstance(k, tuple) else 1) * (2 * base + 1e-6)
        assert d <= bound, (k, d, base)


def test_golden_timesteps_include_both_ends(golden):
    g = golden("denoiser_grad.npz")
    t = g["b3n20_t"].tolist()
    assert 0 in t and 99 in t and len(set(t)) == 3


def test_enable_autograd_is_opt_in_and_not_in_state_dict():
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    assert den.autograd_enabled is False
    keys = set(den.state_dict())
    assert den.enable_autograd() is den and den.autograd_enabled is True
    assert set(den.state_dict()) == keys
    fresh = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    fresh.load_state_dict(den.state_dict(), strict=True)
    assert fresh.autograd_enabled is False
    assert den.enable_autograd(False).autograd_enabled is False


def test_refusals_without_a_device():
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER).enable_autograd()
    x, z = torch.zeros(2, 3, 9), torch.zeros(2, 3, 384)
    with pytest.raises(_native.NativeError, match="CPU"):
        den(x, torch.tensor([1, 2]), z)
    den.enable_autograd(False)
    with pytest.raises(_native.NativeError):
        den(x, torch.tensor([1, 2]), z)
