"""Differentiable Denoiser.forward (Denoiser.enable_autograd, pdb_denoiser_grad_forward / _backward) against the float64 oracle in
tests/denoiser_grad_oracle.py, against p_losses, and against the reference's own fp32 Denoiser (tests/golden/denoiser_grad.npz).

Tolerances follow tests/test_gpu_train.py: per tensor (eps, dL/dx, dL/dz and each of the 108 parameter gradients), the relative L2
distance to the float64 oracle must be at most 5x that of the oracle run with every projection operand truncated to TF32, plus
1e-6."""
import numpy as np
import pytest
import torch

import posediffusion_b200 as pdb
from denoiser_grad_oracle import denoiser_eps, eps_and_grads
from oracle import train_oracle as to
from oracle.make_golden_train import sample_index
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
NAMES = list(syn.denoiser_param_shapes())
# launches of one call: the forward is p_losses' (5 feed kernels, 10 per layer, 2 for the tail).  The full backward is p_losses'
# (17 for the tail, 42 per layer, 10 for _first and the time MLP); dL/dz adds a padded copy, a transpose and a GEMM, dL/dx a padded
# copy, a transpose, a GEMM and the harmonic chain-rule kernel.  Without parameter gradients only the input chain runs: 4 for the
# tail (tail backward, LayerNorm backward, the input gradient's transpose and GEMM) and 14 per layer (3 dropouts, 4 input
# gradients of 2, 2 LayerNorm backwards, attention backward).
FWD_LAUNCHES = 5 + 8 * 10 + 2
BWD_PARAMS, BWD_INPUT_CHAIN, DZ_LAUNCHES, DX_LAUNCHES = 17 + 8 * 42 + 10, 4 + 8 * 14, 3, 4


def make_den(seed=3):
    state = syn.random_denoiser_state(seed, 0.05)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    return den.to(DEV).enable_autograd().eval(), state


def inputs(B, N, seed=0):
    g = torch.Generator().manual_seed(300 + seed)
    x = torch.randn(B, N, 9, generator=g)
    t = torch.randperm(100, generator=g)[:B] if B <= 100 else torch.randint(0, 100, (B,), generator=g)
    z = syn.random_features(B, N, seed)
    ge = torch.randn(B, N, 9, generator=g)
    return x, t, z, ge


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def native(den, x, t, z, ge):
    """eps, parameter gradients (None where a parameter got none), dL/dx, dL/dz of sum(ge * eps) through Denoiser.forward."""
    den.zero_grad(set_to_none=True)
    xx = x.to(DEV).requires_grad_(True)
    zz = z.to(DEV).requires_grad_(True)
    eps = den(xx, t.to(DEV), zz)
    eps.backward(ge.to(DEV))
    grads = {n: (q.grad.clone() if q.grad is not None else None) for n, q in den.named_parameters()}
    return eps.detach(), grads, xx.grad, zz.grad


def as_dict(eps, grads, dx, dz):
    return {"eps": eps, "dx": dx, "dz": dz, **grads}


def check_against_oracle(den, state, x, t, z, ge, p=0.0, seed=None):
    got = as_dict(*native(den, x, t, z, ge))
    ref = as_dict(*eps_and_grads(state, x, t, z, ge, p=p, seed=seed, device=DEV))
    tf = as_dict(*eps_and_grads(state, x, t, z, ge, p=p, seed=seed, tf32="trunc", device=DEV))
    worst = []
    for k in ref:
        d_tf, d_gpu = rel(tf[k], ref[k]), rel(got[k], ref[k])
        worst.append((d_gpu / (5 * d_tf + 1e-6), k, d_gpu, d_tf))
        assert d_gpu <= 5 * d_tf + 1e-6, (k, d_gpu, d_tf)
    worst.sort(reverse=True)
    print(f"B={x.shape[0]} N={x.shape[1]} p={p}: largest error / bound {worst[0][0]:.3f} ({worst[0][1]}: {worst[0][2]:.2e} vs TF32 "
          f"oracle {worst[0][3]:.2e})")
    return got


@pytest.mark.parametrize("B,N", [(2, 5), (3, 20), (1, 64), (51, 10), (170, 3)])
def test_eps_and_all_gradients_against_oracle(B, N):
    """Distinct per-sample timesteps; (1, 64) is the frame limit, (51, 10) and (170, 3) the released recipe's token counts."""
    den, state = make_den()
    x, t, z, ge = inputs(B, N, B + N)
    if B > 1:
        assert len(set(t.tolist())) == B or B > 100
    check_against_oracle(den, state, x, t, z, ge)


def test_dropout_in_train_mode_follows_the_host_masks_and_repeats_bit_identically():
    """The derived bound holds while no ReLU input lies within rounding distance of zero, so that the GPU and both oracle runs
    take the same branches.  At 4 x 33 with torch seed 21 none does; a point where one does (4 x 9 with inputs(4, 9, 1) flips
    one of the tail's ReLUs on the GPU only) moves every gradient upstream of it by a few percent, for the GPU and the
    TF32-emulating oracle alike, but not always in the same run."""
    den, state = make_den()
    den.train()
    x, t, z, ge = inputs(4, 33, 2)
    torch.manual_seed(21)
    seed = int(torch.randint(0, 2**63 - 1, (1,), device=DEV).item())  # the draw the forward makes on the device generator
    torch.manual_seed(21)
    first = check_against_oracle(den, state, x, t, z, ge, p=den.dropout_p, seed=seed)
    torch.manual_seed(21)
    again = as_dict(*native(den, x, t, z, ge))
    assert all(torch.equal(first[k], again[k]) for k in first)
    torch.manual_seed(22)
    other = as_dict(*native(den, x, t, z, ge))
    assert not torch.equal(first["eps"], other["eps"])
    den.eval()
    ev = as_dict(*native(den, x, t, z, ge))
    den.train()
    den.dropout_p, keep = 0.0, den.dropout_p
    zero = as_dict(*native(den, x, t, z, ge))
    den.dropout_p = keep
    assert all(torch.equal(ev[k], zero[k]) for k in ev)
    assert not torch.equal(ev["eps"], first["eps"])


def test_shared_with_p_losses_bit_for_bit():
    """Noise 0, x = x_t, eval mode: |eps| is p_losses' l1 loss, and grad_eps = sign(eps) g gives p_losses' parameter gradients
    for grad_loss = g."""
    den, _ = make_den()
    dif = pdb.GaussianDiffusion(loss_type="l1")
    dif.model = den
    dif = dif.to(DEV).eval()
    x, t, z, g = [v.to(DEV) for v in inputs(3, 7, 2)]
    den.zero_grad(set_to_none=True)
    out = dif.p_losses(x, t, z, torch.zeros_like(x))
    torch.autograd.backward(out["loss"], g)
    want = {n: q.grad.clone() for n, q in den.named_parameters()}
    den.zero_grad(set_to_none=True)
    eps = den(out["x_t"].detach(), t, z)
    assert torch.equal(eps.abs(), out["loss"].detach())
    eps.backward(torch.sign(eps.detach()) * g)
    for n, q in den.named_parameters():
        assert torch.equal(q.grad, want[n]), n


def test_frozen_parameters_run_the_input_chain_only():
    den, _ = make_den()
    ctx = _native.Context.get(DEV)
    x, t, z, ge = inputs(3, 11, 3)
    _, full, dx, dz = native(den, x, t, z, ge)
    assert all(full[n] is not None for n in NAMES)
    den.requires_grad_(False)
    c0 = ctx.launch_count
    _, none, dx2, dz2 = native(den, x, t, z, ge)
    torch.cuda.synchronize()
    assert ctx.launch_count - c0 == FWD_LAUNCHES + BWD_INPUT_CHAIN + DZ_LAUNCHES + DX_LAUNCHES
    assert all(v is None for v in none.values())
    assert torch.equal(dx, dx2) and torch.equal(dz, dz2)
    # dx only
    den.zero_grad(set_to_none=True)
    xx = x.to(DEV).requires_grad_(True)
    c0 = ctx.launch_count
    den(xx, t.to(DEV), z.to(DEV)).backward(ge.to(DEV))
    assert ctx.launch_count - c0 == FWD_LAUNCHES + BWD_INPUT_CHAIN + DX_LAUNCHES
    assert torch.equal(xx.grad, dx)
    # some parameters frozen: all 108 are computed, the frozen ones get none, the others match the full backward
    den.requires_grad_(True)
    den._first.requires_grad_(False)
    _, part, _, _ = native(den, x, t, z, ge)
    for n in NAMES:
        if n.startswith("_first."):
            assert part[n] is None
        else:
            assert torch.equal(part[n], full[n]), n


def test_launch_counts():
    den, _ = make_den()
    ctx = _native.Context.get(DEV)
    x, t, z, ge = [v.to(DEV) for v in inputs(3, 7)]
    counts = [ctx.launch_count]
    eps = den(x.requires_grad_(True), t, z.requires_grad_(True))
    counts.append(ctx.launch_count)
    eps.backward(ge)
    counts.append(ctx.launch_count)
    eps = den(x.detach(), t, z.detach())
    counts.append(ctx.launch_count)
    eps.backward(ge)
    counts.append(ctx.launch_count)
    assert [b - a for a, b in zip(counts, counts[1:])] == [FWD_LAUNCHES, BWD_PARAMS + DZ_LAUNCHES + DX_LAUNCHES, FWD_LAUNCHES, BWD_PARAMS]
    with torch.no_grad():
        c0 = ctx.launch_count
        out = den(x, t, z)
    assert ctx.launch_count - c0 == FWD_LAUNCHES and not out.requires_grad and out.grad_fn is None


def test_gradient_accumulation_and_two_outstanding_graphs():
    den, _ = make_den()
    a = [v.to(DEV) for v in inputs(2, 6, 1)]
    b = [v.to(DEV) for v in inputs(2, 6, 2)]

    def single(v):
        den.zero_grad(set_to_none=True)
        xx = v[0].clone().requires_grad_(True)
        (den(xx, v[1], v[2]) * v[3]).sum().backward()
        return [q.grad.clone() for q in den.parameters()], xx.grad

    (ga, dxa), (gb, dxb) = single(a), single(b)
    den.zero_grad(set_to_none=True)
    xa, xb = a[0].clone().requires_grad_(True), b[0].clone().requires_grad_(True)
    la = (den(xa, a[1], a[2]) * a[3]).sum()
    lb = (den(xb, b[1], b[2]) * b[3]).sum()
    lb.backward()
    la.backward()
    for q, x, y in zip(den.parameters(), ga, gb):
        assert torch.equal(q.grad, x + y)
    assert torch.equal(xa.grad, dxa) and torch.equal(xb.grad, dxb)


def test_inplace_edit_and_second_backward_raise():
    den, _ = make_den()
    x, t, z, ge = [v.to(DEV) for v in inputs(2, 4)]
    eps = den(x, t, z)
    with torch.no_grad():
        den._first.bias.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        eps.backward(ge)
    eps = den(x, t, z)
    eps.backward(ge, retain_graph=True)
    with pytest.raises(RuntimeError, match="already backpropagated"):
        eps.backward(ge)
    eps = den(x, t, z)
    eps.backward(ge)
    with pytest.raises(RuntimeError):
        eps.backward(ge)


def test_refusals():
    den, _ = make_den()
    x, t, z, _ = [v.to(DEV) for v in inputs(2, 65)]
    with pytest.raises(_native.NativeError, match="64 frames"):
        den(x, t, z)
    x, z = x[:, :4].contiguous(), z[:, :4].contiguous()
    with pytest.raises(IndexError):
        den(x, torch.tensor([3, 100], device=DEV), z)
    with pytest.raises(IndexError):
        den(x, torch.tensor(-1, device=DEV), z)
    with pytest.raises(_native.NativeError):
        den(x.cpu(), t, z)
    with pytest.raises(TypeError):
        den(x, t.float(), z)
    # a scalar or one-element t is broadcast to the batch
    one = den(x, torch.tensor(17, device=DEV), z)
    assert torch.equal(one, den(x, torch.full((2,), 17, device=DEV), z))
    assert torch.equal(one, den(x, torch.tensor([17]), z))
    # through the C ABI: the two workspaces are not interchangeable
    ctx = _native.Context.get(DEV)
    params = den.ordered_parameters()
    ws, eps = ctx.denoiser_grad_forward(params, x, t.int(), z, 0.0, 0)
    with pytest.raises(_native.NativeError, match="training forward"):
        ctx.train_backward(params, ws, torch.ones_like(x), None)
    tws, *_ = ctx.train_forward(params, x, t.int(), torch.zeros_like(x), z, 0.0, 0, "l1")
    with pytest.raises(_native.NativeError, match="pdb_denoiser_grad_forward"):
        ctx.denoiser_grad_backward(params, tws, torch.ones_like(x), True)
    ws, _ = ctx.denoiser_grad_forward(params, x, torch.tensor([5, -1], device=DEV, dtype=torch.int32), z, 0.0, 0)
    with pytest.raises(_native.NativeError, match="timestep"):
        ctx.denoiser_grad_backward(params, ws, torch.ones_like(x), True)


def test_flag_off_is_the_inference_kernel():
    den, _ = make_den()
    den.enable_autograd(False)
    x, _, z, _ = [v.to(DEV) for v in inputs(2, 5)]
    t = torch.full((2,), 40, device=DEV)
    x.requires_grad_(True)
    out = den(x, t, z)
    assert out.grad_fn is None and not out.requires_grad
    want = den.native_context().denoiser_forward(x.detach().contiguous(), 40, z)
    assert torch.equal(out, want)
    with pytest.raises(NotImplementedError):
        den(x, torch.tensor([3, 4], device=DEV), z)


def test_against_reference_goldens(golden):
    """GPU vs the reference's own fp32 Denoiser under autograd (eval mode, per-sample t with 0 and 99).  Bound per tensor, as
    tests/test_gpu_train.py's test_against_reference_goldens: 5x the TF32-emulating oracle's distance to float64 plus 2x the fp32
    oracle's, plus 1e-6; four times that for the 64-sample estimate of a fingerprinted tensor."""
    g = golden("denoiser_grad.npz")
    state = syn.random_denoiser_state(int(g["state_seed"][0]), 0.05)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    den = den.to(DEV).enable_autograd().eval()
    r = lambda a, b: float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-30))  # noqa: E731
    for name in ("b2n5", "b3n20", "b1n64"):
        p = f"{name}_"
        x, t, ge = (torch.from_numpy(g[p + k]) for k in ("x", "t", "ge"))
        z = torch.from_numpy(g[p + "z"].astype(np.float32))
        got = {k: v.cpu().numpy() for k, v in as_dict(*native(den, x, t, z, ge)).items()}
        dist = {"eps": r(got["eps"], g[p + "eps"]), "dx": r(got["dx"], g[p + "dx"])}
        for n in NAMES + ["dz"]:
            if p + "grad:" + n in g:
                dist[n] = r(got[n], g[p + "grad:" + n])
            else:
                fp, flat = g[p + "fp:" + n], got[n].astype(np.float64).reshape(-1)
                dist[n] = max(abs(np.linalg.norm(flat) - fp[1]) / fp[1], abs(flat.sum() - fp[0]) / (fp[1] * np.sqrt(flat.size)))
                dist[(n, "samples")] = r(flat[sample_index(flat.size)], fp[2:])
        ref = as_dict(*eps_and_grads(state, x, t, z, ge, device=DEV))
        tf = as_dict(*eps_and_grads(state, x, t, z, ge, tf32="trunc", device=DEV))
        f32 = as_dict(*eps_and_grads(state, x, t, z, ge, dtype=torch.float32, device=DEV))
        base = {k: 5 * rel(tf[k], v) + 2 * rel(f32[k], v) + 1e-6 for k, v in ref.items()}
        worst = 0.0
        for k, d in dist.items():
            bound = base[k[0]] * 4 if isinstance(k, tuple) else base[k]
            worst = max(worst, d / bound)
            assert d <= bound, (name, k, d, bound)
        print(f"{name}: largest distance to the reference fixture / bound {worst:.3f}")


def test_guidance_gradient_through_x0_pred():
    """d ||x_0_pred(x)||^2 / dx with x_0_pred = sqrt(1/abar_t) x - sqrt(1/abar_t - 1) eps(x), through Denoiser.forward and the
    diffuser's schedule buffers, against the same expression on the oracle; parameters frozen (the input chain only)."""
    den, state = make_den()
    den.requires_grad_(False)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    dif = dif.to(DEV)
    x, _, z, _ = inputs(2, 8, 4)
    t = torch.tensor([10, 70])

    def x0_cost(eps_fn, xx, a, b):
        x0 = a.view(-1, 1, 1) * xx - b.view(-1, 1, 1) * eps_fn(xx)
        return (x0 ** 2).sum()

    xx = x.to(DEV).requires_grad_(True)
    td = t.to(DEV)
    cost = x0_cost(lambda v: den(v, td, z.to(DEV)), xx, dif.sqrt_recip_alphas_cumprod[td], dif.sqrt_recipm1_alphas_cumprod[td])
    (got,) = torch.autograd.grad(cost, xx)

    def oracle(tf32):
        params = {k: v.double().to(DEV) for k, v in state.items()}
        xo = x.double().to(DEV).requires_grad_(True)
        a = dif.sqrt_recip_alphas_cumprod[td].double()
        b = dif.sqrt_recipm1_alphas_cumprod[td].double()
        c = x0_cost(lambda v: denoiser_eps(params, v, t, z, tf32=tf32, device=DEV), xo, a, b)
        return torch.autograd.grad(c, xo)[0]

    ref, tf = oracle(None), oracle("trunc")
    d_gpu, d_tf = rel(got, ref), rel(tf, ref)
    print(f"guidance dx: {d_gpu:.2e} vs TF32 oracle {d_tf:.2e}")
    assert d_gpu <= 5 * d_tf + 1e-6
