"""Backbone training path (csrc/api_vit_train.cu) against the float64 autograd of oracle/vit_train_oracle.py.

Tolerances are derived per tensor as in tests/test_gpu_train.py: the oracle runs exactly and with every matrix-product operand
rounded to TF32; the GPU gradient must lie within 5x that run's relative distance to float64 (plus 1e-6)."""
import pytest
import torch

import posediffusion_b200 as pdb
from oracle import train_oracle as to
from oracle import vit_train_oracle as vo
from oracle.dino_vit import DinoViTSmall16, randomize
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
DEFAULT = (1, 1 / 2, 1 / 3)
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)


def make_extractor(seed=11, scales=DEFAULT):
    vit = randomize(DinoViTSmall16(), seed)
    ext = pdb.MultiScaleImageFeatureExtractor(freeze=False, scale_factors=scales)
    ext._net.load_state_dict(vit.state_dict(), strict=True)
    return ext.to(DEV), {k: v.clone() for k, v in vit.state_dict().items()}


def images(n, h=224, w=224, seed=1):
    return torch.rand(n, 3, h, w, generator=torch.Generator().manual_seed(seed))


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp(min=1e-30)).item()


def native_grads(ext, img, g):
    ext.zero_grad(set_to_none=True)
    z = ext(img.to(DEV))
    z.backward(g.to(DEV))
    return z.detach(), {k: p.grad.clone() for k, p in ext._net.named_parameters()}


def check(n, h=224, w=224, scales=DEFAULT):
    ext, state = make_extractor(scales=scales)
    img = images(n, h, w)
    g = torch.randn(n, 384, generator=torch.Generator().manual_seed(7))
    z, grads = native_grads(ext, img, g)
    zr, ref = vo.features_and_grads(state, img, scales, g)
    zt, tf = vo.features_and_grads(state, img, scales, g, tf32=True)
    assert rel(z, zr) <= 5 * rel(zt, zr) + 1e-6, ("z", rel(z, zr), rel(zt, zr))
    worst = []
    for k in ref:
        assert torch.isfinite(grads[k]).all(), k
        d_tf, d_gpu = rel(tf[k].reshape(-1), ref[k].reshape(-1)), rel(grads[k].reshape(-1), ref[k].reshape(-1))
        worst.append((d_gpu / (5 * d_tf + 1e-6), k, d_gpu, d_tf))
    worst.sort(reverse=True)
    print(f"n={n} {h}x{w} scales={len(scales)}: largest gradient error / bound {worst[0][0]:.3f} ({worst[0][1]}: {worst[0][2]:.2e} vs TF32 oracle {worst[0][3]:.2e})")
    bad = [w_ for w_ in worst if w_[0] > 1.0]
    assert not bad, bad[:5]


@pytest.mark.parametrize("n", [1, 2, 7, 21])
def test_gradients_against_oracle(n):
    """n = 1, 2, 7 run the 64-feature GEMM tiles, n = 21 (5544 tokens) the 128-feature tiles for fc1."""
    check(n)


def test_non_square_input_resamples_the_14x14_position_grid():
    check(2, 224, 232)


def test_four_scales_with_upsampling():
    check(1, scales=(1, 1 / 2, 1 / 3, 1.1))


def test_training_z_matches_the_explicit_layernorm_emulation():
    """Section 4.6's bound with the "tf32_ln" emulation: |device - f64| <= 4 |emulation - f64| per image row (plus a floor)."""
    from oracle.vit_f64 import VitF64

    ext, state = make_extractor()
    img = images(3, seed=5)
    z = ext(img.to(DEV)).detach().cpu().double()
    ev = VitF64(state)
    zr, ze = ev.features(img, DEFAULT), ev.features(img, DEFAULT, "tf32_ln")
    err, bound = (z - zr).norm(dim=1), 4 * (ze - zr).norm(dim=1) + 1e-5 * zr.norm(dim=1)
    assert (err <= bound).all(), (err, bound)


def test_two_runs_are_bit_identical_and_second_backward_raises():
    ext, _ = make_extractor()
    img, g = images(3, seed=2), torch.randn(3, 384, generator=torch.Generator().manual_seed(3))
    z1, g1 = native_grads(ext, img, g)
    z2, g2 = native_grads(ext, img, g)
    assert torch.equal(z1, z2) and all(torch.equal(g1[k], g2[k]) for k in g1)
    z = ext(img.to(DEV))
    z.sum().backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="already backpropagated"):
        z.sum().backward()


@pytest.mark.parametrize("h,w,scales,resampled", [(224, 224, DEFAULT, 2), (224, 232, DEFAULT, 3), (224, 224, (1, 1 / 2, 1 / 3, 1.1), 3)])
def test_launch_count_is_the_number_of_kernels_enqueued(h, w, scales, resampled):
    """Forward: one position-table kernel per resampled scale, patchify and position add per scale, the patch GEMM, 8 per block,
    the head.  Backward: 5 for the head, per block 42 plus one attention backward per scale (each linear layer's input, weight and
    bias gradients are 2 + 3 + 2), then the patch weight (3), one position sum per scale and the position gradient."""
    ext, _ = make_extractor(scales=scales)
    ctx = _native.Context.get(DEV)
    params = list(ext._net.parameters())
    k = len(scales)
    before = ctx.launch_count
    ws, z = ctx.vit_train_forward(params, images(2, h, w).to(DEV), scales)
    mid = ctx.launch_count
    ctx.vit_backward(params, ws, torch.ones_like(z))
    after = ctx.launch_count
    assert mid - before == resampled + 2 * k + 1 + 12 * 8 + 1
    assert after - mid == 5 + 12 * (42 + k) + 3 + k + 1


def test_frozen_or_no_grad_calls_take_the_inference_path():
    ext, _ = make_extractor()
    img = images(2).to(DEV)
    with torch.no_grad():
        z0 = ext(img)
    assert z0.grad_fn is None
    frozen = pdb.MultiScaleImageFeatureExtractor(freeze=True).to(DEV)
    frozen._net.load_state_dict(ext._net.state_dict())
    assert torch.equal(frozen(img), z0)
    zt = ext(img)
    assert zt.grad_fn is not None and (zt - z0).abs().max().item() < 2e-2


def make_diffuser(seed=3):
    state = syn.random_denoiser_state(seed, 0.05)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    return dif.to(DEV), state


@pytest.mark.parametrize("B,N", [(2, 5), (6, 20)])
def test_dz_against_oracle_and_parameter_gradients_unchanged(B, N):
    dif, state = make_diffuser()
    den = dif.model
    g = torch.Generator().manual_seed(100 + B)
    x, noise = torch.randn(B, N, 9, generator=g) * 0.5, torch.randn(B, N, 9, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    z = syn.random_features(B, N, 4)
    gl, gx = torch.randn(B, N, 9, generator=g), torch.randn(B, N, 9, generator=g)
    runs = []
    for need in (False, True):
        den.zero_grad(set_to_none=True)
        zd = z.to(DEV).requires_grad_(need)
        loss, x0, _ = den.train_step_forward(x.to(DEV), t.to(DEV), noise.to(DEV), zd, 0.0, 0, "l1")
        torch.autograd.backward([loss, x0], [gl.to(DEV), gx.to(DEV)])
        runs.append(([p.grad.clone() for p in den.parameters()], zd.grad))
    assert runs[0][1] is None and all(torch.equal(a, b) for a, b in zip(runs[0][0], runs[1][0]))

    def oracle_dz(tf32):
        zz = z.double().requires_grad_(True)
        params = {k: v.double() for k, v in state.items()}
        out = to.forward(params, x, t, noise, zz, "l1", None, 0.0, tf32)
        return torch.autograd.grad((out["loss"] * gl.double()).sum() + (out["x_0_pred"] * gx.double()).sum(), zz)[0]

    ref, tf = oracle_dz(None), oracle_dz("trunc")
    assert rel(runs[1][1], ref) <= 5 * rel(tf, ref) + 1e-6, (rel(runs[1][1], ref), rel(tf, ref))


def train_cfg():
    return dict(
        pose_encoding_type="absT_quaR_logFL",
        IMAGE_FEATURE_EXTRACTOR=dict(_target_="models.MultiScaleImageFeatureExtractor", freeze=False),
        DIFFUSER=dict(_target_="models.GaussianDiffusion", beta_schedule="custom"),
        DENOISER=dict(_target_="models.Denoiser", TRANSFORMER=TRANSFORMER, target_dim=9, pivot_cam_onehot=True, z_dim=384, mlp_hidden_dim=128),
    )


def test_facade_trains_all_258_tensors_and_sampling_sees_the_step():
    from types import SimpleNamespace

    torch.manual_seed(0)
    model = pdb.PoseDiffusionModel(**train_cfg())
    ext_state = randomize(DinoViTSmall16(), 11).state_dict()
    model.image_feature_extractor._net.load_state_dict(ext_state, strict=True)
    model.diffuser.model.load_state_dict(syn.random_denoiser_state(3, 0.05), strict=True)
    model = model.to(DEV)
    b, n, rep = 2, 3, 3
    img = torch.rand(b, n, 3, 224, 224, generator=torch.Generator().manual_seed(4)).to(DEV)
    g = torch.Generator().manual_seed(5)
    q = torch.nn.functional.normalize(torch.randn(b * rep * n, 4, generator=g), dim=-1)
    from oracle.shims.pytorch3d.transforms.rotation_conversions import quaternion_to_matrix

    cams = SimpleNamespace(R=quaternion_to_matrix(q).to(DEV), T=torch.randn(b * rep * n, 3, generator=g).to(DEV),
                           focal_length=(1.5 + torch.rand(b * rep * n, 2, generator=g)).to(DEV))
    with torch.no_grad():
        z_before = model(image=img, training=False)["z"]
    assert z_before.grad_fn is None
    opt = torch.optim.AdamW(model.parameters(), lr=1e-4)
    losses = []
    for _ in range(5):
        opt.zero_grad(set_to_none=True)
        loss = model(image=img, gt_cameras=cams, training=True, batch_repeat=rep)["loss"].mean()
        loss.backward()
        params = list(model.parameters())
        assert len(params) == 258
        for name, p in model.named_parameters():
            assert p.grad is not None and torch.isfinite(p.grad).all() and p.grad.abs().max().item() > 0, name
        opt.step()
        losses.append(loss.item())
    assert all(torch.isfinite(torch.tensor(losses)))
    out = model(image=img, training=False)
    assert out["z"].grad_fn is None
    assert not torch.equal(out["z"], z_before)  # the sampler's backbone copy follows the optimizer step
    loss = model(image=img, gt_cameras=cams, training=True, batch_repeat=rep)["loss"].mean()
    loss.backward(retain_graph=True)
    with pytest.raises(RuntimeError, match="already backpropagated"):
        loss.backward()


def test_512_images_gradients_are_finite_reproducible_and_additive_over_images():
    """The released recipe's largest step: 512 images of 224^2 at the default scales (135 168 tokens).  Weight gradients are sums
    over images, so they equal the sum of four 128-image runs (a different dW K length) up to summation order; a dW element is
    one fp32 accumulation over K = 135 168 tokens on the tensor cores, which alone carries about 1e-4 (1.4e-4 measured for the
    patch weight), so the bound is 1e-3."""
    assert _native.vit_train_workspace_bytes(512, 224, 224, DEFAULT) < 40 * 2**30
    ext, _ = make_extractor()
    img = images(512, seed=9).to(DEV)
    g = torch.randn(512, 384, generator=torch.Generator().manual_seed(8)).to(DEV)
    _, full = native_grads(ext, img, g)
    _, again = native_grads(ext, img, g)
    for k in full:
        assert torch.isfinite(full[k]).all(), k
        assert torch.equal(full[k], again[k]), k
    del again
    parts = None
    for i in range(4):
        _, part = native_grads(ext, img[128 * i:128 * (i + 1)], g[128 * i:128 * (i + 1)])
        parts = part if parts is None else {k: parts[k] + part[k] for k in part}
    for k in full:
        assert rel(full[k], parts[k]) <= 1e-3, (k, rel(full[k], parts[k]))
