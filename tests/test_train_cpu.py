"""Training surface without a GPU: the float64 oracle against torch's own modules, the quaternion convention, the host image of
the dropout masks, and the refusals."""
import numpy as np
import pytest
import torch

import posediffusion_b200 as pdb
from oracle import pose_oracle as po
from oracle import train_oracle as to
from oracle.shims.pytorch3d.transforms.rotation_conversions import quaternion_to_matrix
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)


def torch_denoiser(state):
    """The oracle package's nn.TransformerEncoder-based denoiser in float64 and train() mode with every dropout at 0."""
    net = po.build_denoiser(state).double().train()
    for m in net.modules():
        if isinstance(m, torch.nn.Dropout):
            m.p = 0.0
        if isinstance(m, torch.nn.MultiheadAttention):
            m.dropout = 0.0

    def run(x_t, t, z):
        B, N, _ = x_t.shape
        temb = net.time_embed.linear(po.timestep_features(t).double())[:, None, :].expand(-1, N, -1)
        pivot = torch.zeros(B, N, 1, dtype=torch.float64)
        pivot[:, 0] = 1.0
        feed = torch.cat([po.harmonic_features(x_t.float()).double(), temb, z.double(), pivot], dim=-1)
        return net._last(net._trunk(net._first(feed)))

    return net, run


def test_oracle_with_all_ones_masks_matches_torch_transformer_in_train_mode():
    """oracle/train_oracle.py (layer written out, masks injected) vs nn.TransformerEncoder in train() mode at dropout 0."""
    state = syn.random_denoiser_state(2, 0.05)
    net, run = torch_denoiser(state)
    B, N = 3, 6
    g = torch.Generator().manual_seed(0)
    x, noise = torch.randn(B, N, 9, generator=g), torch.randn(B, N, 9, generator=g)
    t = torch.tensor([0, 57, 99])
    z = syn.random_features(B, N, 1)
    ones = {(l, s): torch.ones(shape) for l in range(8)
            for s, shape in ((0, (B, 4, N, N)), (1, (B, N, 512)), (2, (B, N, 1024)), (3, (B, N, 512)))}
    params = {k: v.double() for k, v in state.items()}
    out = to.forward(params, x, t, noise, z, "l2", ones, p=0.0)
    with torch.no_grad():
        eps = run(out["x_t"], t, z)
    torch.testing.assert_close(out["eps"], eps, rtol=0, atol=1e-9)
    sched = po.diffusion_schedule()
    x0 = sched["sqrt_recip_alphas_cumprod"][t].double().view(B, 1, 1) * out["x_t"] - \
        sched["sqrt_recipm1_alphas_cumprod"][t].double().view(B, 1, 1) * eps
    torch.testing.assert_close(out["x_0_pred"], x0, rtol=0, atol=1e-12)
    torch.testing.assert_close(out["loss"], (eps - noise.double()) ** 2, rtol=0, atol=1e-12)


def test_oracle_gradients_match_torch_transformer():
    state = syn.random_denoiser_state(4, 0.05)
    net, run = torch_denoiser(state)
    B, N = 2, 4
    g = torch.Generator().manual_seed(1)
    x, noise = torch.randn(B, N, 9, generator=g), torch.randn(B, N, 9, generator=g)
    t = torch.tensor([3, 80])
    z = syn.random_features(B, N, 2)
    gl = torch.randn(B, N, 9, generator=g)
    out, grads = to.loss_and_grads(state, x, t, noise, z, gl, None, "l1")
    eps = run(out["x_t"], t, z)
    ((eps - noise.double()).abs() * gl.double()).sum().backward()
    named = dict(net.named_parameters())
    for n, g_or in grads.items():
        torch.testing.assert_close(g_or, named[n].grad, rtol=1e-9, atol=1e-12, msg=n)


def test_tf32_rounding_modes():
    x = torch.tensor([1.0 + 2.0 ** -11, 1.0 + 2.0 ** -10 + 2.0 ** -12, -(1.0 + 3 * 2.0 ** -12)], dtype=torch.float64)
    assert to.tf32_round(x, "trunc").tolist() == [1.0, 1.0 + 2.0 ** -10, -1.0]
    assert to.tf32_round(x, "rn").tolist() == [1.0 + 2.0 ** -10, 1.0 + 2.0 ** -10, -(1.0 + 2.0 ** -10)]


def test_quaternion_round_trip_through_the_shim_covers_all_branches():
    g = torch.Generator().manual_seed(3)
    q = torch.randn(400, 4, generator=g, dtype=torch.float64)
    q[:4] = torch.tensor([[1.0, 0.1, 0.05, 0.02], [0.05, 1.0, 0.1, 0.02], [0.02, 0.1, 1.0, 0.05], [0.05, 0.02, 0.1, 1.0]], dtype=torch.float64)
    R = quaternion_to_matrix(q)
    back = to.matrix_to_quaternion(R)
    qn = q / q.norm(dim=-1, keepdim=True)
    qn = torch.where(qn[:, :1] < 0, -qn, qn)
    torch.testing.assert_close(back, qn, rtol=0, atol=1e-12)
    torch.testing.assert_close(quaternion_to_matrix(back), R, rtol=0, atol=1e-12)
    m = R.reshape(-1, 9)
    arg = torch.stack([1 + m[:, 0] + m[:, 4] + m[:, 8], 1 + m[:, 0] - m[:, 4] - m[:, 8], 1 - m[:, 0] + m[:, 4] - m[:, 8],
                       1 - m[:, 0] - m[:, 4] + m[:, 8]], -1)
    assert set(arg.argmax(-1).tolist()) == {0, 1, 2, 3}


@pytest.mark.parametrize("p", [0.1, 0.5])
def test_dropout_mask_keep_fraction_within_binomial_bounds(p):
    n = 1 << 20
    keep = _native.dropout_mask_host(42, 3, 2, 0, n, p)
    mean, sd = n * (1 - p), np.sqrt(n * p * (1 - p))
    assert abs(int(keep.sum()) - mean) < 6 * sd
    # consecutive halves are not correlated with each other
    a, b = keep[: n // 2].astype(np.float64), keep[n // 2:].astype(np.float64)
    assert abs(np.corrcoef(a, b)[0, 1]) < 6 / np.sqrt(n // 2)


def test_dropout_streams_are_distinct_and_offsets_consistent():
    n = 4096
    base = _native.dropout_mask_host(7, 0, 0, 0, n, 0.1)
    others = [_native.dropout_mask_host(8, 0, 0, 0, n, 0.1), _native.dropout_mask_host(7, 1, 0, 0, n, 0.1),
              _native.dropout_mask_host(7, 0, 1, 0, n, 0.1), _native.dropout_mask_host(7 + (1 << 32), 0, 0, 0, n, 0.1)]
    for o in others:
        assert not np.array_equal(base, o)
    assert np.array_equal(_native.dropout_mask_host(7, 0, 0, 1000, 96, 0.1), base[1000:1096])
    assert _native.dropout_mask_host(7, 0, 0, 0, n, 0.0).all()
    with pytest.raises(ValueError):
        _native.dropout_mask_host(7, 8, 0, 0, 4, 0.1)
    with pytest.raises(ValueError):
        _native.dropout_mask_host(7, 0, 0, 0, 4, 1.0)


def test_train_workspace_size():
    small, big = _native.train_workspace_bytes(2, 5), _native.train_workspace_bytes(4, 5)
    assert 0 < small < big
    assert _native.train_workspace_bytes(1, _native.TRAIN_MAX_FRAMES + 1) == 0
    # the released recipe's largest step (51 sequences x 10 frames x 90): saved activations plus backward scratch
    assert _native.train_workspace_bytes(51 * 90, 10) < 12 * 2**30


def test_trainable_feature_extractor_is_refused():
    model = pdb.PoseDiffusionModel(
        pose_encoding_type="absT_quaR_logFL",
        IMAGE_FEATURE_EXTRACTOR={"_target_": "models.MultiScaleImageFeatureExtractor", "freeze": False},
        DIFFUSER={"_target_": "models.GaussianDiffusion", "beta_schedule": "custom"},
        DENOISER={"_target_": "models.Denoiser", "TRANSFORMER": dict(TRANSFORMER, _target_="models.TransformerEncoderWrapper")},
    )
    with pytest.raises(NotImplementedError, match="ViT backward"):
        model(image=torch.zeros(1, 2, 3, 224, 224), gt_cameras=None, training=True)


def test_unknown_loss_type_and_pred_x0_are_refused():
    dif = pdb.GaussianDiffusion(loss_type="huber")
    dif.model = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    with pytest.raises(ValueError, match="invalid loss type"):
        dif.p_losses(torch.zeros(1, 3, 9), torch.zeros(1, dtype=torch.long), torch.zeros(1, 3, 384))
    dif = pdb.GaussianDiffusion(objective="pred_x0")
    dif.model = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    with pytest.raises(NotImplementedError, match="pred_x0"):
        dif.p_losses(torch.zeros(1, 3, 9), torch.zeros(1, dtype=torch.long), torch.zeros(1, 3, 384))


def test_q_sample_matches_the_reference_formula():
    dif = pdb.GaussianDiffusion()
    x, noise = torch.randn(3, 4, 9), torch.randn(3, 4, 9)
    t = torch.tensor([0, 50, 99])
    want = dif.sqrt_alphas_cumprod[t].view(3, 1, 1) * x + dif.sqrt_one_minus_alphas_cumprod[t].view(3, 1, 1) * noise
    assert torch.equal(dif.q_sample(x, t, noise), want)


# ---- the reference's own training step and camera encoding (tests/golden/train.npz, oracle/make_golden_train.py) -------------
from oracle.make_golden_train import CASES as GOLDEN_CASES, sample_index  # noqa: E402


def golden_case(golden, name):
    seqs, frames, rep, loss_type, _ = GOLDEN_CASES[name]
    g = golden("train.npz")
    T = lambda k: torch.from_numpy(g[f"{name}_{k}"])  # noqa: E731
    args = (T("x_start"), T("t"), T("noise"), T("z").repeat(rep, 1, 1), T("gl"), T("gx"), loss_type)
    return g, args


def golden_distance(g, name, values, grads):
    """Per output / gradient tensor: relative L2 distance of `values` / `grads` to the fixture.  For a fingerprinted tensor, key n
    holds the larger of the norm's relative error and |sum error| / (norm sqrt(numel)) (by the triangle and Cauchy-Schwarz
    inequalities both are at most the full tensor's relative L2 distance), and key (n, "samples") the 64 samples' relative L2
    error, which estimates that distance from 64 elements only."""
    p = f"{name}_"
    rel = lambda a, b: float(np.linalg.norm(np.asarray(a, np.float64) - b) / max(np.linalg.norm(b), 1e-30))  # noqa: E731
    out = {k: rel(values[k], g[p + k]) for k in ("x_t", "x_0_pred", "loss")}
    for n, gr in grads.items():
        a = np.asarray(gr, np.float64)
        if p + "grad:" + n in g:
            out[n] = rel(a, g[p + "grad:" + n])
        else:
            fp, flat = g[p + "fp:" + n], a.reshape(-1)
            out[n] = max(abs(np.linalg.norm(flat) - fp[1]) / fp[1], abs(flat.sum() - fp[0]) / (fp[1] * np.sqrt(flat.size)))
            out[(n, "samples")] = rel(flat[sample_index(flat.size)], fp[2:])
    return out


def full_distance(a, b):
    """Relative L2 distance of every tensor of run a to run b (same keys)."""
    return {k: float((a[k].double() - b[k].double()).norm() / b[k].double().norm().clamp(min=1e-30)) for k in b}


@pytest.mark.parametrize("name", sorted(GOLDEN_CASES))
def test_oracle_against_reference_goldens(golden, name):
    """Float64 oracle vs the reference's own fp32 p_losses + Denoiser.  The bound per tensor is derived: twice the distance of the
    same oracle evaluated in float32 from its float64 evaluation (cancelling sums, e.g. LayerNorm gradients, and ReLU inputs near
    zero make some tensors' fp32 error large), plus 1e-6; four times that for the 64-sample estimate of a fingerprinted tensor."""
    g, args = golden_case(golden, name)
    state = syn.random_denoiser_state(int(g["state_seed"][0]), 0.05)
    out, grads = to.loss_and_grads(state, *args)
    o32, g32 = to.loss_and_grads(state, *args, dtype=torch.float32)
    d32 = full_distance({**{k: o32[k] for k in ("x_t", "x_0_pred", "loss")}, **g32},
                        {**{k: out[k] for k in ("x_t", "x_0_pred", "loss")}, **grads})
    got = golden_distance(g, name, {k: out[k].numpy() for k in out}, {n: v.numpy() for n, v in grads.items()})
    for k, d in got.items():
        base = d32[k[0] if isinstance(k, tuple) else k]
        bound = (4 if isinstance(k, tuple) else 1) * (2 * base + 1e-6)
        assert d <= bound, (k, d, base)


def test_camera_goldens_oracle_and_shim_round_trip(golden):
    """The reference's camera_to_pose_encoding (standardised matrix_to_quaternion): every branch, both clamp bounds, flipped
    real parts; the oracle restatement and the shim's quaternion_to_matrix round trip."""
    g = golden("train.npz")
    R, T, focal, want = (torch.from_numpy(g[k]).double() for k in ("cam_R", "cam_T", "cam_focal", "cam_pose"))
    m = R.reshape(-1, 9)
    arg = torch.stack([1 + m[:, 0] + m[:, 4] + m[:, 8], 1 + m[:, 0] - m[:, 4] - m[:, 8], 1 - m[:, 0] + m[:, 4] - m[:, 8],
                       1 - m[:, 0] - m[:, 4] + m[:, 8]], -1)
    assert set(arg.argmax(-1).tolist()) == {0, 1, 2, 3}
    assert (focal < 0.1).any() and (focal > 20).any()
    torch.testing.assert_close(to.camera_to_pose_encoding(R, T, focal), want, rtol=0, atol=1e-6)
    assert (want[:, 3] >= 0).all()
    torch.testing.assert_close(quaternion_to_matrix(want[:, 3:7]), R, rtol=0, atol=2e-6)
