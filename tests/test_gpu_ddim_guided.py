"""Guided DDIM jumps on the GPU: `ddim_sample(..., guided_steps=g')` / `pdb_sample_loop_ddim_guided` /
`pdb_sample_loop_host_matches_ddim` (DESIGN.md "Fewer-step sampling").

Tolerances, as tests/test_gpu_ddim.py states them:
  * each jump's pre-GGS mean, teacher-forced from the device's own state: 4 * d32 + 1e-6 * max(1, max|out|) on the fp32 engine,
    5e-3 * max(1, max|out|) on the tensor-core engine.  GGS is made a no-op there (min_matches so large that every phase is
    dropped at its first evaluation), so the trail holds the jumps' means;
  * with GGS, each guided jump teacher-forced on the generic path (native denoiser, the table row, GGS): 1e-3 * max|x| at 10
    frames, 3e-3 at 20 frames x 380 pairs, the guided-step bounds of DESIGN.md section 2.
"""
import contextlib
import ctypes as C
import io
from functools import partial

import numpy as np
import pytest
import torch

import ddim_guided_oracle as gd
import ddim_oracle as dd
from conftest import load_golden
from oracle.denoiser_f64 import DenoiserF64, bound

import posediffusion_b200 as pdb
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
NO_GGS = dict(min_matches=1e9, verbose=False)  # every GGS phase dropped: the pose stays the jump's mean


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


@contextlib.contextmanager
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


def scenes(B, N, per_pair=16, seed=0):
    return [syn.scene_matches(N, per_pair, seed=seed + b)[0] for b in range(B)]


# ---------------------------------------------------------------------------------------------------
# (a) each guided jump's mean against float64
# ---------------------------------------------------------------------------------------------------
def _jump_means(den, dev, ref, B, N, k, g, gs, eta, tc):
    ctx = den.native_context()
    z = syn.random_features(B, N, 3 * gs + g)
    draws = ddim_draws(k, B, N, eta, 1000 + 10 * gs + g)
    cfg = dict(syn.default_ggs_cfg(), **NO_GGS)
    problems = [ctx.pack_matches(m) for m in scenes(B, N, seed=N)]
    _, trail, stats = ctx.sample_loop_ddim(z.to(dev), draws.to(dev), k + gs, eta, problems, cfg, g, guided_steps=gs)
    trail = trail.cpu()
    assert trail.shape == (1 + k + gs, B, N, 9) and torch.isfinite(trail).all()
    rows = _native.stats_to_numpy(stats)
    assert len(rows) == gs * B and rows["dropped"][:, 0].all()  # GGS left every mean as it was
    worst = 0.0
    for i, (t, s, _c) in enumerate(gd.guided_jumps(g, gs, eta)):
        want, d32 = gd.guided_jump_f64(ref, trail[k + i], t, s, eta, z)
        scale = want.abs().max().item()
        lim = 5e-3 * max(1.0, scale) if tc else bound(d32, scale)
        err = (trail[k + 1 + i].double() - want).abs().max().item()
        assert err <= lim, (i, t, s, err, lim)
        worst = max(worst, err / lim)
    return worst


@pytest.mark.parametrize("g,gs,eta", [(10, 5, 0.0), (10, 3, 0.5), (10, 1, 1.0)])
@pytest.mark.parametrize("flagged", [False, True], ids=["barriers", "flags"])
@pytest.mark.parametrize("N", [2, 10, 20, 128])  # 2 frames stand for 1 (no frame pair to match), on the same 8-token tile
def test_fp32_engine_jump_means_vs_f64(den, dev, ref, N, g, gs, eta, flagged):
    with engine(den.native_context(), "fp32", flagged):
        worst = _jump_means(den, dev, ref, 1, N, 4, g, gs, eta, tc=False)
    print(f"guided jumps fp32 1x{N} g={g} g'={gs} eta={eta}: max err/bound {worst:.3f}")


@pytest.mark.parametrize("g,gs,eta", [(10, 5, 0.0), (10, 2, 0.5)])
@pytest.mark.parametrize("B,N", [(1, 10), (8, 20), (1, 128)])
def test_tc_engine_jump_means_vs_f64(den, dev, ref, B, N, g, gs, eta):
    with engine(den.native_context(), "tf32"):
        worst = _jump_means(den, dev, ref, B, N, 4, g, gs, eta, tc=True)
    print(f"guided jumps tf32 {B}x{N} g={g} g'={gs} eta={eta}: max err/bound {worst:.3f}")


# ---------------------------------------------------------------------------------------------------
# (b) g' = g is pdb_sample_loop_ddim
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("N,eta", [(10, 0.0), (20, 0.5)])
def test_full_guided_steps_bit_identical_to_ddim_entry(den, dev, N, eta):
    ctx = den.native_context()
    k, g = 10, 10
    z = syn.random_features(1, N, 8).to(dev)
    draws = ddim_draws(k, 1, N, eta, 8).to(dev)
    cfg = dict(syn.default_ggs_cfg(), **NO_GGS)  # GGS is not run-to-run bit-reproducible (atomics); dropped phases are
    problems = [ctx.pack_matches(m) for m in scenes(1, N)]
    got, got_trail, _ = ctx.sample_loop_ddim(z, draws, k + g, eta, problems, cfg, g, guided_steps=g)
    want, want_trail = torch.empty_like(got), torch.empty_like(got_trail)
    conf = _native.ggs_config_struct(cfg)
    rc = ctx.lib.pdb_sample_loop_ddim(ctx.handle, z.data_ptr(), draws.data_ptr(), 1, N, k + g, eta, ctx._problem_array(problems), 1,
                                      C.byref(conf), g, want.data_ptr(), want_trail.data_ptr(), None,
                                      C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))
    assert rc == 0
    assert torch.equal(got_trail, want_trail) and torch.equal(got, want)


# ---------------------------------------------------------------------------------------------------
# (c) with GGS: each jump teacher-forced, shapes, the log, and the generic cond_fn path
# ---------------------------------------------------------------------------------------------------
def _scene(frames, per_pair, seed=31):
    """tests/test_gpu_ddim.py's scene: output layer x 0.02, x_T scaled so that the deterministic prefix lands near the scene."""
    state = syn.random_denoiser_state(5, 0.05)
    state["_last.3.weight"] = state["_last.3.weight"] * 0.02
    state["_last.3.bias"] = state["_last.3.bias"] * 0.02
    m, _gt, start = syn.scene_matches(frames, per_pair, seed=seed, ordered=per_pair > 32)
    return state, m, start, syn.random_features(1, frames, seed)


@pytest.mark.parametrize("frames,per_pair,k,gs,tol", [(10, 32, 10, 5, 1e-3), (10, 32, 10, 2, 1e-3), (20, 2048, 20, 5, 3e-3)])
def test_guided_jumps_with_ggs(dev, frames, per_pair, k, gs, tol):
    g = 10
    state, m, start, z = _scene(frames, per_pair)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    dif = dif.to(dev)
    ctx = den.native_context()
    cfg = syn.default_ggs_cfg()
    gain = 1.0
    for _t, _s, c in dd.prefix_steps(k, g, 0.0):
        gain *= c["c1"] * c["a"] + c["c2"]
    draws = (torch.from_numpy(start)[None] / gain).float()[None].to(dev)
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    zd = z.to(dev)
    out = io.StringIO()
    with contextlib.redirect_stdout(out):  # cfg verbose (the default): the reference's log lines
        pose, trail = dif.ddim_sample([1, frames, 9], zd, cond_fn=cond, cond_start_step=g, sampling_timesteps=k + gs, eta=0.0,
                                      draws=draws, guided_steps=gs)
    assert trail.shape == (1 + k + gs, 1, frames, 9) and torch.equal(pose, trail[-1])
    rows = _native.stats_to_numpy(dif.last_ggs_stats)
    assert len(rows) == gs and int(rows["iters"].sum()) == 700 * gs and int(rows["dropped"].sum()) == 0
    starts = [t for t, _s, _c in gd.guided_jumps(g, gs, 0.0)]
    logged = [int(line.split("|")[0].strip()[2:]) for line in out.getvalue().splitlines() if line.startswith("t=")]
    assert logged == [t for t in starts for _ in range(_native.PDB_GGS_PHASES)]
    _, coef = _native.ddim_table(k + gs, g, 0.0, guided_steps=gs)
    quiet = dict(cfg, verbose=False)
    worst = 0.0
    for i, t in enumerate(starts):
        x = trail[k + i].contiguous()
        a, b, c1, c2 = (float(v) for v in coef[k + i, :4])
        eps = ctx.denoiser_forward(x, t, zd)
        want = pdb.geometry_guided_sampling(c1 * (a * x - b * eps) + c2 * x, t, matches_dict=m, GGS_cfg=quiet)
        err = (trail[k + 1 + i] - want).abs().max().item() / want.abs().max().item()
        worst = max(worst, err)
    sampson = [float(rows["sampson"][i][-1]) for i in range(gs)]
    print(f"guided jumps 1x{frames} k={k} g'={gs}: worst jump {worst:.3e} (relative to max|x|); last phase Sampson per jump "
          f"{', '.join(f'{s:.4f}' for s in sampson)}")
    assert worst <= tol, worst
    generic = partial(lambda mean, t, **kw: pdb.geometry_guided_sampling(mean, t, **kw), matches_dict=m, GGS_cfg=quiet)
    pose_g, trail_g = dif.ddim_sample([1, frames, 9], zd, cond_fn=generic, cond_start_step=g, sampling_timesteps=k + gs, eta=0.0,
                                      draws=draws, guided_steps=gs)
    assert trail_g.shape == trail.shape and torch.equal(trail_g[: 1 + k], trail[: 1 + k])  # the same prefix
    err = (pose_g - pose).abs().max().item() / pose.abs().max().item()
    print(f"generic cond_fn vs fused 1x{frames} g'={gs}: {err:.3e}")
    assert err <= tol * gs, err


# ---------------------------------------------------------------------------------------------------
# (d) the host-matches entry, generator use, refusals, the model keyword
# ---------------------------------------------------------------------------------------------------
def test_host_matches_ddim_equals_pack_then_device_entry(den, dev):
    ctx = den.native_context()
    frames, B, k, g, gs, eta = 6, 2, 10, 10, 5, 0.5
    sets = [syn.scene_matches(frames, 48 + 16 * s, seed=71 + s)[0] for s in range(B)]
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=3, min_matches=0, verbose=False)
    z = syn.random_features(B, frames, 72)
    draws = ddim_draws(k, B, frames, eta, 72)
    want, want_trail, want_stats = ctx.sample_loop_ddim(z.to(dev), draws.to(dev), k + gs, eta, [ctx.pack_matches(s) for s in sets],
                                                        cfg, g, guided_steps=gs)
    want, want_trail, want_stats = want.cpu().numpy(), want_trail.cpu().numpy(), _native.stats_to_numpy(want_stats)
    got, got_trail = np.zeros_like(want), np.zeros_like(want_trail)
    got_stats = np.zeros(gs * B, dtype=_native.GGS_STATS_DTYPE)
    ctx.sample_loop_host_matches_ddim(z.numpy(), draws.numpy(), sets, cfg, g, k + gs, eta, got, got_trail, got_stats, guided_steps=gs)
    np.testing.assert_array_equal(got_trail[: 1 + k], want_trail[: 1 + k])  # the prefix: no atomics
    assert np.array_equal(got_stats["iters"], want_stats["iters"]) and (got_stats["iters"] > 0).all()
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-3 * np.abs(want_trail).max())
    with pytest.raises(ValueError):
        ctx.sample_loop_host_matches_ddim(z.numpy(), draws.numpy(), sets, cfg, g, k + gs, eta, got, guided_steps=g + 1)


@pytest.mark.parametrize("eta,k", [(0.0, 10), (0.5, 10), (1.0, 45)])
def test_generator_use(dif, den, dev, eta, k):
    N = 5
    cond = partial(pdb.geometry_guided_sampling, matches_dict=scenes(1, N)[0], GGS_cfg=dict(syn.default_ggs_cfg(), verbose=False))
    z = syn.random_features(1, N, 1).to(dev)
    torch.manual_seed(1234)
    dif.ddim_sample([1, N, 9], z, cond_fn=cond, cond_start_step=10, sampling_timesteps=k + 3, eta=eta, guided_steps=3)
    after = torch.randn(1, N, 9, device=dev)
    torch.manual_seed(1234)
    for _ in range(1 + k if eta > 0 else 1):
        torch.randn(1, N, 9, device=dev)
    assert torch.equal(after, torch.randn(1, N, 9, device=dev))


def test_refusals_launch_nothing(dif, den, dev):
    ctx = den.native_context()
    N = 5
    m = scenes(1, N)[0]
    cfg = dict(syn.default_ggs_cfg(), verbose=False)
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    z = syn.random_features(1, N, 4).to(dev)
    problems = [ctx.pack_matches(m)]
    torch.cuda.synchronize()
    before = ctx.launch_count
    bad = [
        (ValueError, dict(sampling_timesteps=15, guided_steps=5)),  # no guidance
        (ValueError, dict(sampling_timesteps=15, cond_fn=cond, cond_start_step=0, guided_steps=5)),
        (ValueError, dict(sampling_timesteps=15, cond_fn=cond, cond_start_step=10, guided_steps=0)),
        (ValueError, dict(sampling_timesteps=25, cond_fn=cond, cond_start_step=10, guided_steps=11)),
        (ValueError, dict(sampling_timesteps=5, cond_fn=cond, cond_start_step=10, guided_steps=5)),
        (ValueError, dict(sampling_timesteps=96, cond_fn=cond, cond_start_step=10, guided_steps=5)),
        (_native.NativeError, dict(sampling_timesteps=15, cond_fn=cond, cond_start_step=10, guided_steps=5, eta=50.0)),
        (_native.NativeError, dict(sampling_timesteps=15, cond_fn=cond, cond_start_step=10, guided_steps=5, eta=0.5,
                                   draws=torch.zeros(1, 1, N, 9, device=dev))),
    ]
    for exc, kw in bad:
        with pytest.raises(exc):
            dif.ddim_sample([1, N, 9], z, **kw)
    # the library's own checks, past the binding's
    draws = torch.zeros(1, 1, N, 9, device=dev)
    pose, trail = torch.empty(1, N, 9, device=dev), torch.empty(20, 1, N, 9, device=dev)
    conf = _native.ggs_config_struct(cfg)
    stream = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
    for steps, gs, eta in ((15, 0, 0.0), (15, 11, 0.0), (10, 10, 0.0), (15, 5, 50.0), (15, 5, float("nan"))):
        rc = ctx.lib.pdb_sample_loop_ddim_guided(ctx.handle, z.data_ptr(), draws.data_ptr(), 1, N, steps, eta, gs,
                                                 ctx._problem_array(problems), 1, C.byref(conf), 10, pose.data_ptr(),
                                                 trail.data_ptr(), None, stream)
        assert rc == -1, (steps, gs, eta)
    zn, dn = z.cpu().numpy(), draws.cpu().numpy()
    for steps, gs in ((15, 11), (10, 10)):
        with pytest.raises(ValueError):
            ctx.sample_loop_host_matches_ddim(zn, dn, [m], cfg, 10, steps, 0.0, np.zeros((1, N, 9), np.float32), guided_steps=gs)
    with pytest.raises(ValueError, match="DDIM"):  # 1 - abar_s - sigma^2 < 0: refused by the library
        ctx.sample_loop_host_matches_ddim(zn, np.zeros((11, 1, N, 9), np.float32), [m], cfg, 10, 15, 50.0,
                                          np.zeros((1, N, 9), np.float32), guided_steps=5)
    torch.cuda.synchronize()
    assert ctx.launch_count == before


def test_model_forward_keyword(dev, golden_state):
    model = pdb.PoseDiffusionModel(
        pose_encoding_type="absT_quaR_logFL", IMAGE_FEATURE_EXTRACTOR=None,
        DIFFUSER={"_target_": "models.GaussianDiffusion", "beta_schedule": "custom"},
        DENOISER={"_target_": "models.Denoiser", "TRANSFORMER": dict(TRANSFORMER, _target_="models.TransformerEncoderWrapper")},
    ).to(dev)
    model.diffuser.model.load_state_dict(golden_state, strict=True)
    N = 6
    z = syn.random_features(1, N, 6).to(dev)
    cfg = dict(syn.default_ggs_cfg(), **NO_GGS)  # deterministic guided steps
    cond = partial(pdb.geometry_guided_sampling, matches_dict=scenes(1, N)[0], GGS_cfg=cfg)
    torch.manual_seed(5)
    want, _ = model.diffuser.ddim_sample([1, N, 9], z, cond_fn=cond, cond_start_step=10, sampling_timesteps=14, guided_steps=4)
    torch.manual_seed(5)
    cams = model(z=z, training=False, cond_fn=cond, cond_start_step=10, sampling_timesteps=14, guided_steps=4)["pred_cameras"]
    assert torch.equal(cams.T, want[0, :, :3])
    with pytest.raises(ValueError):
        model(z=z, training=False, cond_fn=cond, cond_start_step=10, guided_steps=4)
