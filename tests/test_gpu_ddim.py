"""Fewer-step sampling on the GPU: `GaussianDiffusion.ddim_sample` / `pdb_sample_loop_ddim` (DESIGN.md "Fewer-step sampling").

Tolerances, stated once:
  * one DDIM step, teacher-forced (started from the float64 state): max |device - float64| <= 4 * d32 + 1e-6 * max(1, max|out|)
    on the fp32 engine (oracle/denoiser_f64.py bound; d32 = the fp32 oracle's own distance at that shape and input, from
    tests/ddim_oracle.py), 5e-3 * max(1, max|out|) on the tensor-core engine (TF32 products; tests/test_gpu_tc.py's eps bound);
  * DDIM at k = 100 and eta = 1 against `sample()` with the same draws: on the fp32 engine bit-identical up to the first step whose
    coefficient row differs from the DDPM row in its last bit, and each later step within the teacher-forced bound; on the
    tensor-core engine, whose split-K reductions make two runs of `sample()` itself differ, every step within its bound;
  * the guided tail started from the DDIM prefix's x_{g-1}: the guided-step bounds of DESIGN.md section 2 (1e-3 * max|x| at 10
    frames, 3e-3 at 20 frames x 380 pairs), each step teacher-forced on today's `p_sample` + GGS path.
"""
from contextlib import contextmanager
from functools import partial

import pytest
import torch

import ddim_oracle as dd
from conftest import load_golden
from oracle.denoiser_f64 import DenoiserF64, bound

import posediffusion_b200 as pdb
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
FP32_SHAPES = [(1, 1), (1, 5), (1, 10), (1, 20), (2, 24), (4, 31), (1, 127)]  # every token tile (8, 8, 16, 20, 24, 32, 32)
TC_SHAPES = [(1, 10), (8, 20), (1, 128)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden_state():
    g = load_golden("denoiser.npz")
    return syn.random_denoiser_state(int(g["weight_seed"]), float(g["bias_std"]))


@pytest.fixture(scope="module")
def den(dev, golden_state):
    d = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    d.load_state_dict(golden_state, strict=True)
    return d.to(dev)


@pytest.fixture(scope="module")
def dif(den, dev):
    d = pdb.GaussianDiffusion()
    d.model = den
    return d.to(dev)


@pytest.fixture(scope="module")
def ref(golden_state):
    return DenoiserF64(golden_state)


@contextmanager
def engine(ctx, mode, flagged=False):
    try:
        ctx.set_denoiser_engine(mode)
        ctx.set_denoiser_handover(flagged)
        yield
    finally:
        ctx.set_denoiser_handover(False)
        ctx.set_denoiser_engine("auto")  # the context is shared with every other test module


def ddim_draws(k, B, N, eta, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(1 + k if eta > 0 else 1, B, N, 9, generator=gen)


# ---------------------------------------------------------------------------------------------------
# (a) teacher-forced DDIM steps against float64
# ---------------------------------------------------------------------------------------------------
def _teacher_forced(den, dev, ref, B, N, k, g, eta, tc: bool):
    """Run the prefix once on the device (one launch), then check every step i from the device's own x_{tau} (trail[i]) against
    the float64 step from that same state."""
    ctx = den.native_context()
    z = syn.random_features(B, N, 7 * k + g)
    draws = ddim_draws(k, B, N, eta, 100 * k + 10 * g + int(10 * eta))
    _, trail, _ = ctx.sample_loop_ddim(z.to(dev), draws.to(dev), k + g, eta, None, None, g)
    trail = trail.cpu()
    assert torch.isfinite(trail[: 1 + k]).all()
    assert torch.equal(trail[0], draws[0])
    worst = 0.0
    for i, (t, s, _c) in enumerate(dd.prefix_steps(k, g, eta)):
        noise = draws[1 + i] if eta > 0 else None
        want, _, d32, _ = dd.ddim_step_f64(ref, trail[i], t, s, eta, z, noise)
        scale = want.abs().max().item()
        lim = 5e-3 * max(1.0, scale) if tc else bound(d32, scale)
        err = (trail[1 + i].double() - want).abs().max().item()
        assert err <= lim, (i, t, s, err, lim)
        worst = max(worst, err / lim)
    return worst


@pytest.mark.parametrize("k,g", [(1, 0), (7, 10), (90, 10)])
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("flagged", [False, True], ids=["barriers", "flags"])
@pytest.mark.parametrize("B,N", FP32_SHAPES, ids=[f"{B}x{N}" for B, N in FP32_SHAPES])
def test_fp32_engine_ddim_steps_vs_f64(den, dev, ref, B, N, k, g, eta, flagged):
    if k == 90 and (B * N > 20 or flagged):  # the 90-step prefix at the headline shapes only (float64 reference cost)
        pytest.skip("90-step prefix checked at up to 20 tokens, barrier hand-over")
    with engine(den.native_context(), "fp32", flagged):
        worst = _teacher_forced(den, dev, ref, B, N, k, g, eta, tc=False)
    print(f"DDIM fp32 {B}x{N} k={k} g={g} eta={eta}: max err/bound {worst:.3f}")


@pytest.mark.parametrize("k,g", [(1, 0), (7, 10), (90, 10)])
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("B,N", TC_SHAPES, ids=[f"{B}x{N}" for B, N in TC_SHAPES])
def test_tc_engine_ddim_steps_vs_f64(den, dev, ref, B, N, k, g, eta):
    if k == 90 and B * N > 20:
        pytest.skip("90-step prefix checked at 1 x 10")
    with engine(den.native_context(), "tf32"):
        worst = _teacher_forced(den, dev, ref, B, N, k, g, eta, tc=True)
    print(f"DDIM tf32 {B}x{N} k={k} g={g} eta={eta}: max err/bound {worst:.3f}")


# ---------------------------------------------------------------------------------------------------
# (b) k = 100, eta = 1 is the DDPM loop
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,B,N", [("fp32", 1, 20), ("fp32", 1, 10), ("tf32", 8, 20)])
def test_full_steps_eta_one_against_sample(den, dev, ref, mode, B, N):
    ctx = den.native_context()
    z = syn.random_features(B, N, 3).to(dev)
    draws = syn.predraw_noise(B, N, seed=3).to(dev)  # [101]: slot 100 (t = 0) is zero, unused by both
    _, coef = _native.ddim_table(100, 0, 1.0)
    sched = _native.schedule_table()
    same = [bool((coef[i, :5] == sched[99 - i, :5]).all()) for i in range(100)]
    first_diff = same.index(False) if False in same else 100
    with engine(ctx, mode):
        _, want, _ = ctx.sample_loop(z, draws, None, None, 0)
        _, got, _ = ctx.sample_loop_ddim(z, draws.contiguous(), 100, 1.0, None, None, 0)
    if mode == "fp32":
        assert torch.equal(got[: 1 + first_diff], want[: 1 + first_diff]), first_diff
    else:  # the tensor-core engine's split-K reductions are not run-to-run reproducible: every step against float64 instead
        first_diff = 0
    trail = got.cpu()
    for i in range(first_diff, 100):  # later steps: the DDIM step from the DDIM state within the teacher-forced bound
        t = 99 - i
        want_i, _, d32, _ = dd.ddim_step_f64(ref, trail[i], t, t - 1, 1.0, z.cpu(), draws[1 + i].cpu())
        scale = want_i.abs().max().item()
        lim = bound(d32, scale) if mode == "fp32" else 5e-3 * max(1.0, scale)
        assert (trail[1 + i].double() - want_i).abs().max().item() <= lim, t
    print(f"k=100 eta=1 {mode} {B}x{N}: bit-identical to sample() for the first {first_diff} steps ({sum(same)} equal rows)")


# ---------------------------------------------------------------------------------------------------
# (c) guided runs: the DDIM prefix hands x_{g-1} to today's guided tail
# ---------------------------------------------------------------------------------------------------
def _scene(frames, per_pair=32, seed=31):
    """As tests/test_gpu_denoiser_tiles.py::_scene_loop: output layer x 0.02 (nearly linear unguided dynamics), x_T chosen so that
    the 10 guided steps start near a geometry-consistent scene (here for the DDIM prefix's gain)."""
    state = syn.random_denoiser_state(5, 0.05)
    state["_last.3.weight"] = state["_last.3.weight"] * 0.02
    state["_last.3.bias"] = state["_last.3.bias"] * 0.02
    m, gt, start = syn.scene_matches(frames, per_pair, seed=seed, ordered=per_pair > 32)  # 20 x 2048: cfg3's 380 ordered pairs
    z = syn.random_features(1, frames, seed)
    return state, m, start, z


@pytest.mark.parametrize("frames,per_pair,k,tol", [(10, 32, 10, 1e-3), (20, 2048, 20, 3e-3)])
def test_guided_ddim_tail_equals_todays_guided_path(dev, frames, per_pair, k, tol):
    g = 10
    state, m, start, z = _scene(frames, per_pair)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    dif = dif.to(dev)
    ctx = den.native_context()
    cfg = syn.default_ggs_cfg()
    cfg.update(verbose=False)
    # x_T such that the deterministic prefix (eps ~ 0: x_s = (c1 a + c2) x_t) lands near the scene
    gain = 1.0
    for _t, _s, c in dd.prefix_steps(k, g, 0.0):
        gain *= c["c1"] * c["a"] + c["c2"]
    draws = (torch.from_numpy(start)[None] / gain).float()[None]
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    zd = z.to(dev)
    pose, trail = dif.ddim_sample([1, frames, 9], zd, cond_fn=cond, cond_start_step=g, sampling_timesteps=k + g, eta=0.0,
                                  draws=draws.to(dev))
    assert trail.shape == (1 + k + g, 1, frames, 9) and torch.equal(pose, trail[-1])
    rows = _native.stats_to_numpy(dif.last_ggs_stats)
    assert len(rows) == g * 1
    assert int(rows["iters"].sum()) == 7000 and int(rows["dropped"].sum()) == 0
    assert (trail[k][0].cpu() - torch.from_numpy(start)).abs().max().item() < 0.5  # the guided steps start near the scene
    worst = 0.0
    for i, t in enumerate(reversed(range(g))):
        want, _ = dif.p_sample(trail[k + i].contiguous(), t, zd, cond_fn=cond, cond_start_step=g)
        err = (trail[k + 1 + i] - want).abs().max().item() / want.abs().max().item()
        worst = max(worst, err)
    print(f"guided DDIM 1x{frames} k={k}: worst guided step {worst:.3e} (relative to max|x|)")
    assert worst <= tol, worst
    # the generic cond_fn path (native prefix, Python guided loop) against the fused one
    generic = partial(lambda mean, t, **kw: pdb.geometry_guided_sampling(mean, t, **kw), matches_dict=m, GGS_cfg=cfg)
    pose_g, trail_g = dif.ddim_sample([1, frames, 9], zd, cond_fn=generic, cond_start_step=g, sampling_timesteps=k + g, eta=0.0,
                                      draws=draws.to(dev))
    assert torch.equal(trail_g[: 1 + k], trail[: 1 + k])  # the same prefix
    err = (pose_g - pose).abs().max().item() / pose.abs().max().item()
    print(f"generic cond_fn vs fused 1x{frames}: {err:.3e}")
    assert err <= tol * g, err


# ---------------------------------------------------------------------------------------------------
# (d) generator use and refusals
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("eta,k", [(0.0, 10), (0.5, 10), (1.0, 45)])
def test_generator_use(dif, dev, eta, k):
    z = syn.random_features(1, 5, 1).to(dev)
    torch.manual_seed(1234)
    dif.ddim_sample([1, 5, 9], z, sampling_timesteps=k, eta=eta)
    after = torch.randn(1, 5, 9, device=dev)
    torch.manual_seed(1234)
    for _ in range(1 + k if eta > 0 else 1):
        torch.randn(1, 5, 9, device=dev)
    assert torch.equal(after, torch.randn(1, 5, 9, device=dev))


def test_ddim_draws_are_the_loop_input(dif, dev):
    z = syn.random_features(1, 5, 2).to(dev)
    torch.manual_seed(99)
    pose_a, trail_a = dif.ddim_sample([1, 5, 9], z, sampling_timesteps=20, eta=0.5)
    torch.manual_seed(99)
    draws = dif.ddim_draws((1, 5, 9), dev, 20, 0.5)
    pose_b, trail_b = dif.ddim_sample([1, 5, 9], z, sampling_timesteps=20, eta=0.5, draws=draws)
    assert torch.equal(trail_a, trail_b) and torch.equal(trail_a[0], draws[0])


def test_refusals_launch_nothing(dif, den, dev):
    ctx = den.native_context()
    z = syn.random_features(1, 5, 4).to(dev)
    draws = syn.predraw_noise(1, 5, seed=4).to(dev)
    pose0, trail0 = dif.p_sample_loop([1, 5, 9], z, draws=draws)
    before = ctx.launch_count
    bad = [
        (ValueError, dict(sampling_timesteps=0)),
        (ValueError, dict(sampling_timesteps=101)),
        (ValueError, dict(sampling_timesteps=10, eta=-0.5)),
        (ValueError, dict(sampling_timesteps=10, eta=float("nan"))),
        (_native.NativeError, dict(sampling_timesteps=10, eta=0.0, draws=torch.zeros(11, 1, 5, 9, device=dev))),
        (_native.NativeError, dict(sampling_timesteps=10, eta=0.5, draws=torch.zeros(1, 1, 5, 9, device=dev))),
        (_native.NativeError, dict(sampling_timesteps=10, eta=50.0)),  # 1 - abar_s - sigma^2 < 0: refused by the library
    ]
    for exc, kw in bad:
        with pytest.raises(exc):
            dif.ddim_sample([1, 5, 9], z, **kw)
    z129 = torch.zeros(1, 129, 384, device=dev)
    with pytest.raises(_native.NativeError, match="PDB_MAX_FRAMES"):
        ctx.sample_loop_ddim(z129, torch.zeros(1, 1, 129, 9, device=dev), 10, 0.0, None, None, 0)
    torch.cuda.synchronize()
    assert ctx.launch_count == before
    pose1, trail1 = dif.p_sample_loop([1, 5, 9], z, draws=draws)
    assert torch.equal(pose1, pose0) and torch.equal(trail1, trail0)


def test_model_forward_keyword(dev, golden_state):
    """PoseDiffusionModel.forward(..., sampling_timesteps=k, eta=...) samples with ddim_sample; None keeps sample()."""
    model = pdb.PoseDiffusionModel(
        pose_encoding_type="absT_quaR_logFL", IMAGE_FEATURE_EXTRACTOR=None,
        DIFFUSER={"_target_": "models.GaussianDiffusion", "beta_schedule": "custom"},
        DENOISER={"_target_": "models.Denoiser", "TRANSFORMER": dict(TRANSFORMER, _target_="models.TransformerEncoderWrapper")},
    ).to(dev)
    model.diffuser.model.load_state_dict(golden_state, strict=True)
    z = syn.random_features(1, 6, 6).to(dev)
    for steps, eta in ((10, 0.0), (20, 0.5)):
        torch.manual_seed(5)
        want, _ = model.diffuser.ddim_sample([1, 6, 9], z, sampling_timesteps=steps, eta=eta)
        torch.manual_seed(5)
        cams = model(z=z, training=False, sampling_timesteps=steps, eta=eta)["pred_cameras"]
        assert torch.equal(cams.T, want[0, :, :3])
    torch.manual_seed(5)
    want, _ = model.diffuser.sample([1, 6, 9], z)
    torch.manual_seed(5)
    assert torch.equal(model(z=z, training=False)["pred_cameras"].T, want[0, :, :3])
