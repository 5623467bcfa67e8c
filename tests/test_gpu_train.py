"""Native training step (csrc/api_train.cu) against the float64 restatement in oracle/train_oracle.py.

Tolerances are derived per tensor: the oracle is run twice, exactly and with every projection operand rounded to TF32 the way the
tensor cores read it; the GPU result must lie within 5x that run's relative distance to float64 (plus 1e-6), measured as
||got - f64|| / ||f64|| per output or gradient tensor."""
import numpy as np
import pytest
import torch

import posediffusion_b200 as pdb
from oracle import train_oracle as to
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
NAMES = list(syn.denoiser_param_shapes())


def make_diffuser(seed=3, loss_type="l1"):
    state = syn.random_denoiser_state(seed, 0.05)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion(loss_type=loss_type)
    dif.model = den
    return dif.to(DEV), state


def inputs(B, N, seed=0):
    g = torch.Generator().manual_seed(100 + seed)
    x = torch.randn(B, N, 9, generator=g) * 0.5
    noise = torch.randn(B, N, 9, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    z = syn.random_features(B, N, seed)
    return x, t, noise, z


def host_masks(seed, B, N, p):
    masks = {}
    for l in range(8):
        for site, shape in ((0, (B, 4, N, N)), (1, (B, N, 512)), (2, (B, N, 1024)), (3, (B, N, 512))):
            n = int(np.prod(shape))
            masks[(l, site)] = torch.from_numpy(_native.dropout_mask_host(seed, l, site, 0, n, p).reshape(shape).astype(np.float64))
    return masks


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def native_step(dif, x, t, noise, z, gl, gx0, p, seed):
    den = dif.model
    den.zero_grad(set_to_none=True)
    loss, x0, x_t = den.train_step_forward(x.to(DEV), t.to(DEV), noise.to(DEV), z.to(DEV), p, seed, dif.loss_type)
    torch.autograd.backward([loss, x0], [gl.to(DEV), gx0.to(DEV)])
    return {"loss": loss, "x_0_pred": x0, "x_t": x_t}, {n: q.grad.clone() for n, q in den.named_parameters()}


def check_against_oracle(dif, state, B, N, p=0.0, seed=0, loss_type="l1", repeat=1):
    x, t, noise, z = inputs(B, N, B + N)
    if repeat > 1:
        z = z[: B // repeat].repeat(repeat, 1, 1)
    g = torch.Generator().manual_seed(7)
    gl, gx0 = torch.randn(B, N, 9, generator=g), torch.randn(B, N, 9, generator=g)
    masks = host_masks(seed, B, N, p) if p > 0 else None
    out, grads = native_step(dif, x, t, noise, z, gl, gx0, p, seed)
    ref, rgrads = to.loss_and_grads(state, x, t, noise, z, gl, gx0, loss_type, masks, p)
    tf, tgrads = to.loss_and_grads(state, x, t, noise, z, gl, gx0, loss_type, masks, p, tf32="trunc")
    worst = []
    for k in ("x_t", "x_0_pred", "loss"):
        bound = 5 * rel(tf[k], ref[k]) + 1e-6
        assert rel(out[k], ref[k]) <= bound, (k, rel(out[k], ref[k]), bound)
    for n in NAMES:
        d_tf, d_gpu = rel(tgrads[n], rgrads[n]), rel(grads[n], rgrads[n])
        worst.append((d_gpu / (5 * d_tf + 1e-6), n, d_gpu, d_tf))
        assert d_gpu <= 5 * d_tf + 1e-6, (n, d_gpu, d_tf)
    worst.sort(reverse=True)
    print(f"B={B} N={N} p={p}: largest gradient error / bound {worst[0][0]:.3f} ({worst[0][1]}: {worst[0][2]:.2e} vs TF32 oracle {worst[0][3]:.2e})")


def test_tf32_operand_rounding_is_truncation():
    """The projections' TF32 convention, checked once on pdb_debug_tc_linear: operands with low mantissa bits set are truncated."""
    ctx = _native.Context.get(DEV)
    g = torch.Generator().manual_seed(5)
    x = torch.randn(256, 512, generator=g)
    w = torch.randn(128, 512, generator=g) * 0.05
    y = ctx.tc_linear(x.to(DEV), w.to(DEV)).cpu().double()
    errs = {m: (y - to.tf32_round(x.double(), m) @ to.tf32_round(w.double(), m).T).abs().max().item() for m in ("trunc", "rn")}
    print("tc_linear vs TF32 emulation:", errs)
    assert errs["trunc"] < errs["rn"] / 4, errs


@pytest.mark.parametrize("B,N", [(2, 5), (3, 20)])
@pytest.mark.parametrize("loss_type", ["l1", "l2"])
def test_small_shapes_against_oracle(B, N, loss_type):
    dif, state = make_diffuser(loss_type=loss_type)
    check_against_oracle(dif, state, B, N, loss_type=loss_type)


@pytest.mark.parametrize("B,N", [(51, 10), (10, 50), (170, 3)])
def test_training_shapes_batch_repeat_2(B, N):
    """The released recipe's sequence shapes with batch_repeat 2: the features of B sequences repeated twice (z.repeat(2, 1, 1),
    as PoseDiffusionModel does), with 2B poses, timesteps and noise draws."""
    dif, state = make_diffuser()
    check_against_oracle(dif, state, 2 * B, N, repeat=2)


@pytest.mark.parametrize("B,N", [(2, 5), (4, 33)])
def test_dropout_masks_from_host_function(B, N):
    dif, state = make_diffuser()
    check_against_oracle(dif, state, B, N, p=0.1, seed=0x1234_5678_9ABC)


def test_eval_mode_equals_dropout_zero_and_repeats_are_bit_identical():
    dif, _ = make_diffuser()
    x, t, noise, z = [v.to(DEV) for v in inputs(3, 7)]
    den = dif.model
    den.train()
    runs = []
    for seed in (11, 11, 12):
        torch.manual_seed(seed)
        den.zero_grad(set_to_none=True)
        out = dif.p_losses(x, t, z, noise)
        out["loss"].mean().backward()
        runs.append((out["loss"].detach().clone(), [q.grad.clone() for q in den.parameters()]))
    assert torch.equal(runs[0][0], runs[1][0]) and all(torch.equal(a, b) for a, b in zip(runs[0][1], runs[1][1]))
    assert not torch.equal(runs[0][0], runs[2][0])
    den.eval()
    ev = dif.p_losses(x, t, z, noise)["loss"]
    den.train()
    den.dropout_p, keep = 0.0, den.dropout_p
    zero = dif.p_losses(x, t, z, noise)["loss"]
    den.dropout_p = keep
    assert torch.equal(ev, zero)
    assert not torch.equal(ev, runs[0][0])


def test_two_outstanding_graphs_and_grad_accumulation():
    dif, _ = make_diffuser()
    den = dif.model.eval()
    a = [v.to(DEV) for v in inputs(2, 6, 1)]
    b = [v.to(DEV) for v in inputs(2, 6, 2)]

    def single(v):
        den.zero_grad(set_to_none=True)
        dif.p_losses(v[0], v[1], v[3], v[2])["loss"].sum().backward()
        return [q.grad.clone() for q in den.parameters()]

    ga, gb = single(a), single(b)
    den.zero_grad(set_to_none=True)
    la = dif.p_losses(a[0], a[1], a[3], a[2])["loss"].sum()
    lb = dif.p_losses(b[0], b[1], b[3], b[2])["loss"].sum()
    lb.backward()
    la.backward()
    for q, x, y in zip(den.parameters(), ga, gb):
        assert torch.equal(q.grad, x + y)


def test_parameter_changed_between_forward_and_backward_raises():
    dif, _ = make_diffuser()
    x, t, noise, z = [v.to(DEV) for v in inputs(2, 4)]
    loss = dif.p_losses(x, t, z, noise)["loss"].sum()
    with torch.no_grad():
        dif.model._first.bias.add_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        loss.backward()


def test_reference_rng_draw_order():
    dif, _ = make_diffuser()
    pose = torch.randn(4, 6, 9, device=DEV)
    z = torch.randn(4, 6, 384, device=DEV)
    torch.manual_seed(123)
    out = dif(pose, z=z)
    torch.manual_seed(123)
    t = torch.randint(0, 100, (4,), device=DEV).long()
    noise = torch.randn_like(pose)
    assert torch.equal(out["t"], t) and torch.equal(out["noise"], noise)
    assert set(out) == {"loss", "noise", "x_0_pred", "x_t", "t"}
    assert out["loss"].shape == (4, 6, 9)
    torch.testing.assert_close(out["x_t"], dif.q_sample(pose, t, noise), rtol=0, atol=1e-6)


def test_loss_type_and_objective_refusals():
    dif, _ = make_diffuser()
    x, t, noise, z = [v.to(DEV) for v in inputs(1, 3)]
    dif.loss_type = "huber"
    with pytest.raises(ValueError):
        dif.p_losses(x, t, z, noise)
    dif.loss_type = "l1"
    dif.objective = "pred_x0"
    with pytest.raises(NotImplementedError):
        dif.p_losses(x, t, z, noise)


def _cameras(n, seed=0):
    g = torch.Generator().manual_seed(seed)
    q = torch.randn(n, 4, generator=g)
    # one rotation per matrix_to_quaternion branch: identity-like, and 180-degree-like turns about x, y and z
    q[:4] = torch.tensor([[1.0, 0.1, 0.05, 0.02], [0.05, 1.0, 0.1, 0.02], [0.02, 0.1, 1.0, 0.05], [0.05, 0.02, 0.1, 1.0]])
    rot = pdb.pose_encoding_to_camera(torch.cat([torch.zeros(n, 3), q, torch.zeros(n, 2)], 1).to(DEV)).R.cpu()
    T = torch.randn(n, 3, generator=g)
    focal = torch.exp(torch.randn(n, 2, generator=g) * 2.0)
    focal[0] = torch.tensor([0.01, 50.0])  # both clamp bounds
    return rot, T, focal


def test_camera_to_pose_encoding_against_oracle_and_round_trip():
    rot, T, focal = _cameras(64)
    cams = pdb.PerspectiveCameras(focal_length=focal.to(DEV), R=rot.to(DEV), T=T.to(DEV))
    got = pdb.camera_to_pose_encoding(cams).cpu()
    want = to.camera_to_pose_encoding(rot.double(), T.double(), focal.double())
    torch.testing.assert_close(got.double(), want, rtol=0, atol=2e-6)
    branches = set(torch.stack([1 + rot[:, 0, 0] + rot[:, 1, 1] + rot[:, 2, 2], 1 + rot[:, 0, 0] - rot[:, 1, 1] - rot[:, 2, 2],
                                1 - rot[:, 0, 0] + rot[:, 1, 1] - rot[:, 2, 2], 1 - rot[:, 0, 0] - rot[:, 1, 1] + rot[:, 2, 2]], -1)
                   .argmax(-1).tolist())
    assert branches == {0, 1, 2, 3}
    assert (got[:, 3] >= 0).all()
    back = pdb.pose_encoding_to_camera(got.to(DEV))
    torch.testing.assert_close(back.R.cpu(), rot, rtol=0, atol=2e-6)


def test_pose_diffusion_model_training_dict():
    model = pdb.PoseDiffusionModel(
        pose_encoding_type="absT_quaR_logFL", IMAGE_FEATURE_EXTRACTOR=None,
        DIFFUSER={"_target_": "models.GaussianDiffusion", "beta_schedule": "custom"},
        DENOISER={"_target_": "models.Denoiser", "TRANSFORMER": dict(TRANSFORMER, _target_="models.TransformerEncoderWrapper")},
    ).to(DEV)
    model.train()
    B, N, rep = 2, 5, 3
    rot, T, focal = _cameras(B * rep * N, 4)
    cams = pdb.PerspectiveCameras(focal_length=focal.to(DEV), R=rot.to(DEV), T=T.to(DEV))
    z = torch.randn(B, N, 384, device=DEV)
    torch.manual_seed(0)
    out = model(gt_cameras=cams, z=z, training=True, batch_repeat=rep)
    assert set(out) == {"loss", "noise", "x_0_pred", "x_t", "t", "pred_cameras"}
    assert out["loss"].shape == (B * rep, N, 9) and len(out["pred_cameras"]) == B * rep * N
    out["loss"].mean().backward()
    assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in model.diffuser.model.parameters())
    torch.nn.utils.clip_grad_norm_(model.parameters(), 1.0)


def test_sampler_picks_up_stepped_weights():
    dif, _ = make_diffuser()
    den = dif.model
    x, t, noise, z = [v.to(DEV) for v in inputs(2, 5)]
    draws = syn.predraw_noise(2, 5, seed=1).to(DEV)
    before, _ = dif.p_sample_loop([2, 5, 9], z, draws=draws)
    opt = torch.optim.AdamW(den.parameters(), lr=1e-3)
    dif.p_losses(x, t, z, noise)["loss"].mean().backward()
    opt.step()
    after, _ = dif.p_sample_loop([2, 5, 9], z, draws=draws)
    fresh = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    fresh.load_state_dict({k: v.detach().cpu() for k, v in den.state_dict().items()})
    dif2 = pdb.GaussianDiffusion()
    dif2.model = fresh
    want, _ = dif2.to(DEV).p_sample_loop([2, 5, 9], z, draws=draws)
    assert not torch.equal(before, after)
    assert torch.equal(after, want)


def test_five_adamw_steps_against_oracle():
    """Dropout 0, pre-drawn t / noise; AdamW (lr 1e-4) on the native gradients vs on the float64 oracle's.  AdamW divides each
    gradient by its running magnitude, so elements whose gradient is near the TF32 noise move by +-lr either way: the bound is the
    deviation of the TF32-emulating oracle's run from the float64 run."""
    dif, state = make_diffuser()
    den = dif.model.eval()
    opt = torch.optim.AdamW(den.parameters(), lr=1e-4)
    refs = {m: {k: v.double().clone().requires_grad_(True) for k, v in state.items()} for m in (None, "trunc")}
    ropts = {m: torch.optim.AdamW([r[n] for n in NAMES], lr=1e-4) for m, r in refs.items()}
    for step in range(5):
        x, t, noise, z = inputs(4, 8, step)
        opt.zero_grad()
        dif.p_losses(x.to(DEV), t.to(DEV), z.to(DEV), noise.to(DEV))["loss"].mean().backward()
        opt.step()
        for m, r in refs.items():
            ropts[m].zero_grad()
            to.forward(r, x, t, noise, z, tf32=m)["loss"].mean().backward()
            ropts[m].step()
    got = dict(den.named_parameters())
    flat = lambda d: torch.cat([(d[n].detach().double().cpu() - state[n].double()).flatten() for n in NAMES])  # noqa: E731
    dev, dev_tf = rel(flat(got), flat(refs[None])), rel(flat(refs["trunc"]), flat(refs[None]))
    print(f"five AdamW steps: relative deviation of the update from the float64 run {dev:.3e} (TF32-emulating oracle {dev_tf:.3e})")
    assert dev < 2 * dev_tf + 1e-3


def test_out_of_range_timesteps_are_refused():
    dif, _ = make_diffuser()
    x, t, noise, z = [v.to(DEV) for v in inputs(2, 4)]
    with pytest.raises(IndexError):
        dif.p_losses(x, torch.tensor([3, 100], device=DEV), z, noise)
    # through the C ABI the forward flags the bad timestep in its workspace (no synchronisation) and the backward refuses it
    ctx = _native.Context.get(DEV)
    params = dif.model.ordered_parameters()
    ws, *_ = ctx.train_forward(params, x, torch.tensor([-1, 5], device=DEV, dtype=torch.int32), noise, z, 0.0, 0, "l1")
    with pytest.raises(_native.NativeError, match="timestep"):
        ctx.train_backward(params, ws, torch.ones_like(x), None)


def test_launch_count_is_the_number_of_kernels_enqueued():
    """Forward: 5 feed kernels, 10 per layer, 2 for the tail.  Backward: 17 for the tail, 42 per layer (each linear layer's input,
    weight and bias gradients are 2 + 3 + 2), 10 for _first and the time MLP; dL/dz adds a padded copy, a transpose and a GEMM."""
    dif, _ = make_diffuser()
    ctx = _native.Context.get(DEV)
    params = dif.model.ordered_parameters()
    x, t, noise, z = [v.to(DEV) for v in inputs(3, 7)]
    counts = [ctx.launch_count]
    ws, *_ = ctx.train_forward(params, x, t.int(), noise, z, 0.1, 5, "l1")
    counts.append(ctx.launch_count)
    ctx.train_backward(params, ws, torch.ones_like(x), None)
    counts.append(ctx.launch_count)
    ctx.train_backward(params, ws, torch.ones_like(x), None, grad_z=torch.empty_like(z))
    counts.append(ctx.launch_count)
    assert [b - a for a, b in zip(counts, counts[1:])] == [5 + 8 * 10 + 2, 17 + 8 * 42 + 10, 17 + 8 * 42 + 10 + 3]


# ---- the reference's own training step and camera encoding (tests/golden/train.npz, oracle/make_golden_train.py) -------------
from oracle.make_golden_train import CASES as GOLDEN_CASES, sample_index  # noqa: E402


def _golden_distance(g, name, values, grads):
    """As tests/test_train_cpu.py: relative L2 distance per tensor; fingerprinted tensors give (norm / sum bound, 64 samples)."""
    p = f"{name}_"
    r = lambda a, b: float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-30))  # noqa: E731
    out = {k: r(values[k], g[p + k]) for k in ("x_t", "x_0_pred", "loss")}
    for n, gr in grads.items():
        a = np.asarray(gr, np.float64)
        if p + "grad:" + n in g:
            out[n] = r(a, g[p + "grad:" + n])
        else:
            fp, flat = g[p + "fp:" + n], a.reshape(-1)
            out[n] = max(abs(np.linalg.norm(flat) - fp[1]) / fp[1], abs(flat.sum() - fp[0]) / (fp[1] * np.sqrt(flat.size)))
            out[(n, "samples")] = r(flat[sample_index(flat.size)], fp[2:])
    return out


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_against_reference_goldens(golden, name):
    """GPU vs the reference's own fp32 p_losses + Denoiser (dropout 0, injected t / noise; one case with batch_repeat 3).  Bound per
    tensor: 5x the TF32-emulating oracle's distance to float64 plus 2x the fp32 oracle's (the fixture is itself fp32), plus 1e-6;
    four times that for the 64-sample estimate of a fingerprinted tensor."""
    seqs, frames, rep, loss_type, _ = GOLDEN_CASES[name]
    g = golden("train.npz")
    T = lambda k: torch.from_numpy(g[f"{name}_{k}"])  # noqa: E731
    x, t, noise, gl, gx = T("x_start"), T("t"), T("noise"), T("gl"), T("gx")
    z = T("z").repeat(rep, 1, 1)
    state = syn.random_denoiser_state(int(g["state_seed"][0]), 0.05)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion(loss_type=loss_type)
    dif.model = den
    dif = dif.to(DEV).eval()
    out = dif.p_losses(x.to(DEV), t.to(DEV), z.to(DEV), noise.to(DEV))
    torch.autograd.backward([out["loss"], out["x_0_pred"]], [gl.to(DEV), gx.to(DEV)])
    grads = {n: q.grad.cpu().numpy() for n, q in den.named_parameters()}
    got = _golden_distance(g, name, {k: out[k].detach().cpu().numpy() for k in ("x_t", "x_0_pred", "loss")}, grads)
    args = (x, t, noise, z, gl, gx, loss_type)
    ref, rg = to.loss_and_grads(state, *args)
    tf, tg = to.loss_and_grads(state, *args, tf32="trunc")
    f32, g32 = to.loss_and_grads(state, *args, dtype=torch.float32)
    both = lambda o, gr: {**{k: o[k] for k in ("x_t", "x_0_pred", "loss")}, **gr}  # noqa: E731
    base = {k: 5 * rel(both(tf, tg)[k], v) + 2 * rel(both(f32, g32)[k], v) + 1e-6 for k, v in both(ref, rg).items()}
    worst = 0.0
    for k, d in got.items():
        bound = base[k[0]] * 4 if isinstance(k, tuple) else base[k]
        worst = max(worst, d / bound)
        assert d <= bound, (k, d, bound)
    print(f"{name}: largest distance to the reference fixture / bound {worst:.3f}")


def test_camera_to_pose_encoding_against_reference_goldens(golden):
    """pdb_camera_to_pose vs the reference's camera_to_pose_encoding: all four matrix_to_quaternion branches, negative real
    parts made positive, focal lengths beyond both clamp bounds."""
    g = golden("train.npz")
    R, T, focal, want = (torch.from_numpy(g[k]) for k in ("cam_R", "cam_T", "cam_focal", "cam_pose"))
    cams = pdb.PerspectiveCameras(focal_length=focal.to(DEV), R=R.to(DEV), T=T.to(DEV))
    got = pdb.camera_to_pose_encoding(cams).cpu()
    torch.testing.assert_close(got, want, rtol=0, atol=1e-6)
