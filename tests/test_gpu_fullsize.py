"""GPU parity at the BASELINE sizes: the CUDA path (through the C ABI) against the CPU oracle, not against itself.

Sizes (SURVEY.md section 8): config 3 = 20 frames x 380 ordered pairs x 2048 = 778 240 matches (the shared-memory-resident
slice path), config 5 = 80 frames x 6320 pairs x 4096 = 25 886 720 matches (the bulk-async ring path, ~340 rounds per warp).
Scenes are geometry-consistent (`syn.scene_matches`), so that about half of the matches are valid and every frame receives
gradient.  Both match-stream layouts run.

Tolerances, stated once:
  * gradient: 1e-3 * max|grad| against the float64 closed form (`oracle.sampson_f64.sampson_closed_form_f64_large`).  fp32 is
    the limit at this size: the reference's own operator sequence in fp32 (`po.sampson_terms` + autograd) is 3.3e-4 * max|grad|
    away from the float64 result on the config-3 scene, the CUDA path 3.3e-4 as well (measured, round 2);
  * valid count: validity is an fp32 comparison `err < sampson_max` on an error computed with a different (fused) operation
    order than the reference's, so a match whose float64 error lies within 1e-5 (relative) of the threshold may flip.  The
    oracle counts those matches (`band`); the device count must lie within max(2, band) of the oracle's;
  * clamped mean error (`sampson_to_print`): 1e-4 relative; mean valid error: 1e-4 relative;
  * five-phase GGS pose after 35 inner iterations at config-3 size: 3e-5 * max|pose| against `po.geometry_guided_sampling`;
  * full T=100 loop, N=20, GGS on (700 inner iterations per guided step): every step teacher-forced on the ORACLE's trajectory,
    unguided steps 3e-5 * max|x|, guided steps 3e-3 * max|x| (700 clipped SGD steps amplify summation-order differences:
    1.65e-3 measured with 20 frames x 380 pairs, round 2; the 6-frame run of test_ggs_long_run_vs_oracle stays within 1e-3).
"""
from functools import partial

import numpy as np
import pytest
import torch

from oracle import pose_oracle as po
from oracle import sampson_f64 as s64

import posediffusion_b200 as pdb
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def ctx(dev):
    return _native.Context.get(dev)


def pack(ctx, m, layout):
    before = ctx.ggs_layout
    ctx.set_ggs_layout(layout)
    try:
        return ctx.pack_matches(m)
    finally:
        ctx.set_ggs_layout(before)  # the context is shared with every other test module


@pytest.fixture(scope="module")
def cfg3_scene():
    m, gt, start = syn.scene_matches(20, 2048, seed=77)
    return m, start, s64.sampson_closed_form_f64_large(start, m)


def check_eval(ctx, dev, m, start, ref, layout, flags=(True, True, True)):
    pm = pack(ctx, m, layout)
    grad, sc, _, _ = ctx.sampson_eval(pm, torch.from_numpy(start).to(dev), *flags)
    n_valid = int(round(sc[1].item()))
    assert abs(n_valid - ref["n_valid"]) <= max(2, ref["band"]), (n_valid, ref["n_valid"], ref["band"])
    gmax = np.abs(ref["grad"]).max()
    np.testing.assert_allclose(grad.cpu().numpy(), ref["grad"], rtol=0, atol=1e-3 * gmax)
    np.testing.assert_allclose(sc[2].item(), ref["logged"], rtol=1e-4)
    np.testing.assert_allclose(sc[0].item(), ref["loss"], rtol=1e-4)


@pytest.mark.parametrize("layout", ["plain", "paired"])
def test_sampson_eval_vs_f64_oracle_at_config3_size(ctx, dev, cfg3_scene, layout):
    """778 240 matches: one CTA per SM, ~184 rounds per CTA on 132 SMs staged in shared memory (the path the headline bench runs)."""
    m, start, ref = cfg3_scene
    assert len(m["kp1"]) == 380 * 2048 and ref["n_valid"] > 300000
    check_eval(ctx, dev, m, start, ref, layout)


@pytest.mark.parametrize("layout", ["plain", "paired"])
def test_sampson_eval_flags_vs_f64_oracle_at_config3_size(ctx, dev, cfg3_scene, layout):
    m, start, _ = cfg3_scene
    for flags in ((True, False, False), (False, True, False), (False, False, True)):
        ref = s64.sampson_closed_form_f64_large(start, m, *flags)
        check_eval(ctx, dev, m, start, ref, layout, flags)


@pytest.mark.parametrize("layout", ["plain", "paired"])
def test_sampson_eval_vs_f64_oracle_at_config5_size(ctx, dev, layout):
    """25 886 720 matches (414 MB): every warp streams ~340 rounds through its bulk-async ring."""
    m, gt, start = syn.scene_matches(80, 4096, seed=78)
    assert len(m["kp1"]) == 6320 * 4096
    ref = s64.sampson_closed_form_f64_large(start, m)
    assert ref["n_valid"] > 5_000_000
    check_eval(ctx, dev, m, start, ref, layout)


@pytest.mark.parametrize("layout", ["plain", "paired"])
def test_ggs_five_phases_vs_oracle_at_config3_size(ctx, dev, cfg3_scene, layout):
    """pdb_ggs with iter_num = 5 (10 + 5 + 5 + 5 + 10 inner iterations) against the oracle's geometry_guided_sampling."""
    m, start, _ = cfg3_scene
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=5, verbose=False)
    pose = torch.from_numpy(start)[None].to(dev).clone()
    stats = _native.stats_to_numpy(ctx.ggs([pack(ctx, m, layout)], pose, cfg))[0]
    log = []
    want = po.geometry_guided_sampling(torch.from_numpy(start)[None], 5, m, cfg, log=log)
    assert list(stats["iters"]) == [e["iters"] for e in log] == [10, 5, 5, 5, 10]
    assert int(stats["dropped"].sum()) == 0
    np.testing.assert_allclose(pose[0].cpu().numpy(), want[0].numpy(), rtol=0, atol=3e-5 * np.abs(want).max().item())
    np.testing.assert_allclose(stats["sampson"], [e["sampson"] for e in log], rtol=1e-3)


def test_full_loop_ggs_on_teacher_forced_on_oracle_trajectory(dev):
    """T = 100, N = 20, GGS on with the default 700 inner iterations per guided step.  The oracle runs the whole loop on the
    CPU (small match set so that its 7 000 inner iterations finish in seconds); every one of the 100 steps of the CUDA path is
    then started from the oracle's state and compared with the oracle's next state.

    Operating point: with random weights the sampler's trajectory has nothing to do with any scene, the guided steps then see a
    handful of borderline-valid matches and 700 clipped SGD steps amplify one validity flip into percent-level differences
    (measured 4.8e-2, round 2) -- in the reference as much as here.  The test therefore puts the loop where a trained model
    would put it: the output layer of the (otherwise random) denoiser is scaled by 0.02, so the unguided dynamics are nearly
    linear, x_{t-1} ~ k_t x_t, and x_T is chosen such that the state entering the first guided step is the perturbed
    ground-truth pose of a geometry-consistent scene (most matches valid, as in test_ggs_long_run_vs_oracle)."""
    frames = 20
    state = syn.random_denoiser_state(5, 0.05)
    state["_last.3.weight"] = state["_last.3.weight"] * 0.02
    state["_last.3.bias"] = state["_last.3.bias"] * 0.02
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    dif = dif.to(dev)
    net = po.build_denoiser(state)
    sched = po.diffusion_schedule()
    m, gt, start = syn.scene_matches(frames, 24, seed=31)
    cfg = syn.default_ggs_cfg()
    cfg.update(verbose=False)
    z = syn.random_features(1, frames, 31)
    gain = 1.0
    for t in range(99, 9, -1):  # eps ~ 0: x_{t-1} = (c1_t a_t + c2_t) x_t
        gain *= float(sched["posterior_mean_coef1"][t] * sched["sqrt_recip_alphas_cumprod"][t] + sched["posterior_mean_coef2"][t])
    draws = 1e-3 * syn.predraw_noise(1, frames, seed=31)
    draws[0] = torch.from_numpy(start)[None] / gain
    cond_o = partial(po.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    log = []
    _, ref = po.p_sample_loop(net, sched, z, draws, partial(po.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg, log=log), 10)
    assert torch.isfinite(ref).all()
    assert all(e["iters"] in (100, 200) and not e["dropped"] for e in log) and len(log) == 50  # 10 guided steps x 5 phases, no early exit
    assert (ref[90][0] - torch.from_numpy(start)).abs().max().item() < 0.5  # the guided steps start near the scene
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    zd = z.to(dev)
    worst_unguided = worst_guided = 0.0
    for t in range(99, -1, -1):
        k = 99 - t
        x = ref[k].to(dev).contiguous()
        if t < 10:
            got, _ = dif.p_sample(x, t, zd, cond_fn=cond, cond_start_step=10)
        else:
            got, _, _ = den.native_context().p_sample(x, t, zd, draws[1 + k].to(dev).contiguous())
        err = (got.cpu() - ref[k + 1]).abs().max().item() / ref[k + 1].abs().max().item()
        if t < 10:
            worst_guided = max(worst_guided, err)
        else:
            worst_unguided = max(worst_unguided, err)
    assert worst_unguided <= 3e-5, worst_unguided
    assert worst_guided <= 3e-3, worst_guided
