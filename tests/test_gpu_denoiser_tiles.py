"""The sampler at the frame counts it runs: every token-tile width of the fp32 denoiser kernel, both engines, both stage
hand-overs, the frame-count limits, and the 10-frame evaluation loop, against a float64 evaluation of the same network.

The fp32 persistent kernel (csrc/denoiser.cuh) is compiled for token tiles TS in {8, 16, 20, 24, 32}; pick_token_tile
(csrc/api_sampler.cu) takes the width that pads B*N least and the wider one on a tie.  Below 128 tokens the auto engine uses it,
at 128 and above the wgmma/TMA engine (TF32 products).

Tolerances, stated once (oracle/denoiser_f64.py):
  * fp32 engine, eps and one DDPM step: max |device - float64| <= 4 * d32 + 1e-6 * max(1, max|out|), d32 = the fp32 oracle's
    own distance to float64 at that shape and input (1e-7 .. 4e-7 for eps), and never above the fixture bounds of
    tests/test_gpu_parity.py (3e-5 on eps).  Err / bound, largest per tile, measured on an NVIDIA H100 80GB HBM3 (700 W
    power limit) with the golden weights: DESIGN.md section 2;
  * eps of one sequence alone and as a member of batches that pick TS 20, 32, 8, 24: bit-identical (every output has one owner,
    and no summation order depends on TS);
  * tensor-core engine: 5e-3 absolute on eps against float64 (test_gpu_tc.py), and clearly above the fp32 bound, so that the
    engine switch at 128 tokens is observed;
  * 10-frame guided loop (T = 100, 10 guided steps of 700 inner GGS iterations, 45 pairs): teacher-forced on the oracle's
    trajectory, unguided steps 3e-5 * max|x|, guided steps 1e-3 * max|x| (see the test).
"""
from contextlib import contextmanager
from functools import partial

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import pose_oracle as po
from oracle.denoiser_f64 import DenoiserF64, bound

import posediffusion_b200 as pdb
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)

# (B, N) per token tile: edge frame counts, 0..7 padded rows, sequences that straddle tile boundaries
SWEEP = {
    8: [(1, 1), (1, 2), (1, 3), (1, 7), (5, 10)],
    16: [(1, 9), (1, 10), (1, 12), (1, 16)],
    20: [(1, 17), (1, 33), (2, 10), (1, 97)],
    24: [(1, 21), (1, 24), (1, 48), (1, 65), (3, 7), (12, 10)],
    32: [(1, 31), (1, 32), (1, 64), (1, 96), (1, 127), (3, 10), (4, 31)],
}
STEPS = (99, 37, 0)


def token_tile(tokens):
    """pick_token_tile of csrc/api_sampler.cu."""
    return min((8, 16, 20, 24, 32), key=lambda c: ((tokens + c - 1) // c * c, -c))


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


def inputs(B, N, seed):
    gen = torch.Generator().manual_seed(seed)
    return torch.randn(B, N, 9, generator=gen), torch.randn(B, N, 384, generator=gen)


_f64 = {}


def eps_f64(ref, B, N, seed, t):
    key = (B, N, seed, t)
    if key not in _f64:
        x, z = inputs(B, N, seed)
        _f64[key] = ref.noise_f64(x, t, z)
    return _f64[key]


def forward(den, dev, x, t, z):
    return den(x.to(dev), torch.full((x.shape[0],), t, dtype=torch.long, device=dev), z.to(dev)).cpu()


# ---------------------------------------------------------------------------------------------------
# (a) fp32 engine: every token tile against float64
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flagged", [False, True], ids=["barriers", "flags"])
@pytest.mark.parametrize("ts,B,N", [(ts, B, N) for ts, shapes in SWEEP.items() for B, N in shapes],
                         ids=[f"ts{ts}-{B}x{N}" for ts, shapes in SWEEP.items() for B, N in shapes])
def test_fp32_engine_every_token_tile_vs_f64(den, dev, ref, ts, B, N, flagged):
    assert token_tile(B * N) == ts
    x, z = inputs(B, N, 100 * B + N)
    ctx = den.native_context()
    worst = 0.0
    with engine(ctx, "fp32", flagged):
        for t in STEPS:
            got = forward(den, dev, x, t, z)
            want, d32 = eps_f64(ref, B, N, 100 * B + N, t)
            assert torch.isfinite(got).all()
            err = (got.double() - want).abs().max().item()
            assert bound(d32) <= 3e-5
            assert err <= bound(d32), (t, err, d32)
            worst = max(worst, err / bound(d32))
    print(f"fp32 engine TS {ts} {B}x{N} {'flags' if flagged else 'barriers'}: max err/bound {worst:.3f}")


# ---------------------------------------------------------------------------------------------------
# (b) a sequence's eps does not depend on the token tile its batch picks
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flagged", [False, True], ids=["barriers", "flags"])
def test_eps_of_a_sequence_independent_of_token_tile(den, dev, flagged):
    """One 10-frame sequence alone (TS 16) and as a member of batches of 2, 3, 5 and 12 sequences (TS 20, 32, 8, 24), placed so
    that with TS 8 and 24 it straddles a tile boundary: eps bit-identical."""
    x, z = inputs(1, 10, 7)
    ctx = den.native_context()
    with engine(ctx, "fp32", flagged):
        alone = forward(den, dev, x, 42, z)
        for B, at, ts in ((2, 1, 20), (3, 1, 32), (5, 2, 8), (12, 7, 24)):
            assert token_tile(B * 10) == ts
            xb, zb = inputs(B, 10, 70 + B)
            xb[at], zb[at] = x[0], z[0]
            got = forward(den, dev, xb, 42, zb)
            assert torch.equal(got[at], alone[0]), (B, ts, (got[at] - alone[0]).abs().max().item())


# ---------------------------------------------------------------------------------------------------
# (c) both stage hand-overs give the same trajectory at the new widths
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N", [(1, 10), (1, 24), (1, 32), (12, 10)])
def test_handover_modes_bit_identical_at_every_width(den, dev, B, N):
    """As test_denoiser_handover_modes_bit_identical (tests/test_gpu_parity.py), at TS 16, 24, 32 and 24 (12 sequences): a whole
    100-step unguided trajectory in one launch; the flagged mode twice, the second launch over the first one's stale words."""
    ctx = den.native_context()
    z = syn.random_features(B, N, 9).to(dev)
    draws = syn.predraw_noise(B, N, seed=9).to(dev)
    with engine(ctx, "fp32", False):
        pose_a, trail_a, _ = ctx.sample_loop(z, draws, None, None, 0)
    with engine(ctx, "fp32", True):
        pose_b, trail_b, _ = ctx.sample_loop(z, draws, None, None, 0)
        pose_c, trail_c, _ = ctx.sample_loop(z, draws, None, None, 0)
    assert torch.isfinite(trail_a).all()
    assert torch.equal(trail_a, trail_b) and torch.equal(pose_a, pose_b)
    assert torch.equal(trail_a, trail_c) and torch.equal(pose_a, pose_c)


# ---------------------------------------------------------------------------------------------------
# (d) 10-frame sampling steps
# ---------------------------------------------------------------------------------------------------
def test_p_sample_10_frames_every_timestep_vs_f64(den, dev, ref):
    """Teacher-forced p_sample at 1 x 10 (TS 16) for t = 99 .. 0, each step started from the float64 trajectory.  x_{t-1} and x0
    within 4 * d32 + 1e-6 * max|.| of float64; x_{t-1} also within the fixture bound of test_p_sample_teacher_forced_vs_reference."""
    N = 10
    z = syn.random_features(1, N, 10)
    draws = syn.predraw_noise(1, N, seed=10)
    ctx = den.native_context()
    zd = z.to(dev)
    x = draws[0].clone()
    worst = 0.0
    for t in range(99, -1, -1):
        k = 99 - t
        noise = draws[1 + k]
        pred, _, x0 = ctx.p_sample(x.to(dev), t, zd, None if t == 0 else noise.to(dev))
        want, want_x0, d32, d32_x0 = ref.p_sample_f64(x, t, z, noise)
        scale, scale_x0 = want.abs().max().item(), want_x0.abs().max().item()
        b_t = float(ref.sched["sqrt_recipm1_alphas_cumprod"][t])
        assert bound(d32, scale) <= 2e-5 * scale + 1e-5 and bound(d32_x0, scale_x0) <= 1e-5 * scale_x0 + 3e-5 * b_t
        err = (pred.cpu().double() - want).abs().max().item()
        err_x0 = (x0.cpu().double() - want_x0).abs().max().item()  # x0 = a_t x - b_t eps: the eps error times b_t (up to 12.4)
        assert err <= bound(d32, scale), (t, err, d32)
        assert err_x0 <= bound(d32_x0, scale_x0), (t, err_x0, d32_x0)
        worst = max(worst, err / bound(d32, scale), err_x0 / bound(d32_x0, scale_x0))
        x = want.float()
    print(f"p_sample 1x10, 100 steps: max err/bound {worst:.3f}")


def test_one_launch_equals_chain_of_single_steps_10_frames(den, dev):
    """sample_loop without guidance (steps 99 .. 0 in one persistent launch, z projection computed once) == 100 single-step
    p_sample launches, each fed the loop's own previous state: bit for bit (test_emulated_multi_step_launch_equals_single_steps
    checks the same on the CPU)."""
    N = 10
    ctx = den.native_context()
    z = syn.random_features(1, N, 11).to(dev)
    draws = syn.predraw_noise(1, N, seed=11).to(dev)
    pose, trail, _ = ctx.sample_loop(z, draws, None, None, 0)
    assert torch.equal(trail[0], draws[0]) and torch.equal(pose, trail[100])
    for t in range(99, -1, -1):
        k = 99 - t
        one, _, _ = ctx.p_sample(trail[k].contiguous(), t, z, None if t == 0 else draws[1 + k].contiguous())
        assert torch.equal(one, trail[k + 1]), (t, (one - trail[k + 1]).abs().max().item())


# ---------------------------------------------------------------------------------------------------
# (e) the evaluation-shaped guided loop: 10 frames, GGS on, cond_start_step 10
# ---------------------------------------------------------------------------------------------------
def _scene_loop(frames):
    """The operating point of test_full_loop_ggs_on_teacher_forced_on_oracle_trajectory (tests/test_gpu_fullsize.py): output
    layer x 0.02 so that the unguided dynamics are nearly linear, x_T chosen so that the first guided step starts at the perturbed
    ground truth of a geometry-consistent scene."""
    state = syn.random_denoiser_state(5, 0.05)
    state["_last.3.weight"] = state["_last.3.weight"] * 0.02
    state["_last.3.bias"] = state["_last.3.bias"] * 0.02
    sched = po.diffusion_schedule()
    m, gt, start = syn.scene_matches(frames, 32, seed=31, ordered=False)
    z = syn.random_features(1, frames, 31)
    gain = 1.0
    for t in range(99, 9, -1):  # eps ~ 0: x_{t-1} = (c1_t a_t + c2_t) x_t
        gain *= float(sched["posterior_mean_coef1"][t] * sched["sqrt_recip_alphas_cumprod"][t] + sched["posterior_mean_coef2"][t])
    draws = 1e-3 * syn.predraw_noise(1, frames, seed=31)
    draws[0] = torch.from_numpy(start)[None] / gain
    return state, sched, m, start, z, draws


def test_guided_loop_10_frames_teacher_forced_on_oracle_trajectory(dev):
    """T = 100, N = 10, 45 unordered pairs x 32 matches, GGS on with the default 700 inner iterations per guided step,
    cond_start_step 10.  The oracle runs the whole loop on the CPU; each of the 100 CUDA steps starts from the oracle's state.
    Guided-step bound 1e-3 * max|x|: 700 clipped SGD steps amplify summation-order differences; measured 4.8e-4 here on an
    NVIDIA H100 80GB HBM3 (700 W power limit), against 1.65e-3 with 20 frames x 380 pairs and a 3e-3 bound (DESIGN.md
    section 2)."""
    frames = 10
    state, sched, m, start, z, draws = _scene_loop(frames)
    assert len(m["kp1"]) == 45 * 32
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    dif = dif.to(dev)
    net = po.build_denoiser(state)
    cfg = syn.default_ggs_cfg()
    cfg.update(verbose=False)
    log = []
    _, ref = po.p_sample_loop(net, sched, z, draws, partial(po.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg, log=log), 10)
    assert torch.isfinite(ref).all()
    assert all(e["iters"] in (100, 200) and not e["dropped"] for e in log) and len(log) == 50  # 10 guided steps x 5 phases
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
    print(f"guided loop 1x10: worst unguided {worst_unguided:.3e}, worst guided {worst_guided:.3e} (relative to max|x|)")
    assert worst_unguided <= 3e-5, worst_unguided
    assert worst_guided <= 1e-3, worst_guided


def test_fused_host_entry_10_frames_equals_pack_then_loop(dev):
    """pdb_sample_loop_host_matches (the end-to-end entry: packing overlapped with the unguided prefix) at 1 x 10 with the
    evaluation's settings == pdb_matches_pack + pdb_sample_loop_host, and its unguided prefix == the device-buffer loop that
    GaussianDiffusion.p_sample_loop runs (test_host_matches_entry_equals_pack_then_host_entry at 6 frames).  The guided steps
    differ between two launches only by the GGS atomics' summation order, which 10 free-running steps of 700 iterations amplify:
    final poses within 5e-3 * max|x| (1.3e-3 measured on an NVIDIA H100 80GB HBM3, 700 W power limit)."""
    frames = 10
    state, _, m, _, z, draws = _scene_loop(frames)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    dif = dif.to(dev)
    ctx = den.native_context()
    cfg = syn.default_ggs_cfg()
    cfg.update(verbose=False)
    zn, dn = z.numpy(), draws.numpy()
    want, want_trail = np.zeros((1, frames, 9), np.float32), np.zeros((101, 1, frames, 9), np.float32)
    want_stats = np.zeros(10, dtype=_native.GGS_STATS_DTYPE)
    ctx.sample_loop_host(zn, dn, [ctx.pack_matches(m)], cfg, 10, want, want_trail, want_stats)
    got, got_trail = np.zeros_like(want), np.zeros_like(want_trail)
    got_stats = np.zeros_like(want_stats)
    ctx.sample_loop_host_matches(zn, dn, [m], cfg, 10, got, got_trail, got_stats)
    np.testing.assert_array_equal(got_trail[:91], want_trail[:91])  # unguided part: no atomics
    assert np.array_equal(got_stats["iters"], want_stats["iters"]) and (got_stats["iters"] > 0).all()
    assert int(got_stats["dropped"].sum()) == 0
    scale = np.abs(want_trail).max()
    np.testing.assert_allclose(got, want, rtol=0, atol=5e-3 * scale)
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    pose_d, trail_d = dif.p_sample_loop([1, frames, 9], z.to(dev), cond, 10, draws=draws.to(dev))
    np.testing.assert_array_equal(trail_d[:91].cpu().numpy(), want_trail[:91])
    np.testing.assert_allclose(pose_d.cpu().numpy(), want, rtol=0, atol=5e-3 * scale)


# ---------------------------------------------------------------------------------------------------
# (f) tensor-core engine at the same frame counts, and the switch at 128 tokens
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,B,N", [("tf32", 1, 10), ("tf32", 2, 24), ("tf32", 1, 65), ("tf32", 1, 127), ("tf32", 1, 128),
                                      ("auto", 1, 128), ("auto", 13, 10), ("auto", 1, 127)])
def test_tensor_core_engine_vs_f64(den, dev, ref, mode, B, N):
    """TF32 products: 5e-3 absolute on eps against float64 (test_gpu_tc.py), and more than 10x the fp32 engine's bound, so that
    the result shows which engine ran: auto mode switches at 128 tokens (1 x 128, 13 x 10) and stays on the fp32 kernel at 127."""
    x, z = inputs(B, N, 300 + 100 * B + N)
    ctx = den.native_context()
    with engine(ctx, mode):
        got = forward(den, dev, x, 23, z)
    want, d32 = ref.noise_f64(x, 23, z)
    err = (got.double() - want).abs().max().item()
    print(f"{mode} {B}x{N}: err {err:.3e}, fp32 bound {bound(d32):.3e}")
    if mode == "auto" and B * N < 128:
        assert err <= bound(d32), err
        return
    assert 10 * bound(d32) < err < 5e-3, err


# ---------------------------------------------------------------------------------------------------
# (g) frame-count limits: 128 frames through both engines and the loop, 129 refused
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("flagged", [False, True], ids=["barriers", "flags"])
def test_fp32_engine_128_frames_vs_f64(den, dev, ref, flagged):
    """PDB_MAX_FRAMES = 128 on the fp32 kernel (forced; TS 32, 4 tiles): attention covers at most 4 passes of 32 keys, so the
    last key row of the longest sequence is computed and checked, not just accepted."""
    assert token_tile(128) == 32
    x, z = inputs(1, 128, 128)
    ctx = den.native_context()
    with engine(ctx, "fp32", flagged):
        for t in STEPS:
            got = forward(den, dev, x, t, z)
            want, d32 = eps_f64(ref, 1, 128, 128, t)
            err = (got.double() - want).abs().max().item()
            assert err <= bound(d32) <= 3e-5, (t, err, d32)


@pytest.mark.parametrize("mode", ["auto", "fp32"])
def test_sample_loop_128_frames(den, dev, ref, mode):
    """sample_loop at 1 x 128 frames (auto: the tensor-core engine; fp32 forced: the persistent kernel, TS 32): the trajectory
    is finite and steps 99, 50 and 0 of it are within the engine's bound of a float64 step from the loop's own state
    (tensor cores: the 5e-3 eps bound times c1_t b_t, the factor by which eps enters x_{t-1})."""
    N = 128
    ctx = den.native_context()
    z = syn.random_features(1, N, 12)
    draws = syn.predraw_noise(1, N, seed=12)
    with engine(ctx, mode):
        pose, trail, _ = ctx.sample_loop(z.to(dev), draws.to(dev), None, None, 0)
    trail = trail.cpu()
    assert torch.isfinite(trail).all() and torch.equal(pose.cpu(), trail[100])
    for t in (99, 50, 0):
        k = 99 - t
        want, _, d32, _ = ref.p_sample_f64(trail[k], t, z, draws[1 + k])
        scale = want.abs().max().item()
        err = (trail[k + 1].double() - want).abs().max().item()
        if mode == "fp32":
            tol = bound(d32, scale)
        else:
            tol = float(ref.sched["posterior_mean_coef1"][t] * ref.sched["sqrt_recipm1_alphas_cumprod"][t]) * 5e-3 + 1e-5 * scale
        assert err <= tol, (t, err, tol)


def test_129_frames_refused_and_context_still_usable(den, dev):
    """129 frames > PDB_MAX_FRAMES: NativeError (PDB_ERR_LIMIT) from Denoiser.forward, p_sample and sample_loop in every engine
    mode, before anything runs; the next call on the same context computes what it computed before."""
    ctx = den.native_context()
    x, z = inputs(1, 10, 5)
    before = forward(den, dev, x, 50, z)
    xb, zb = (v.to(dev) for v in inputs(1, 129, 6))
    draws = syn.predraw_noise(1, 129, seed=6).to(dev)
    t = torch.full((1,), 50, dtype=torch.long, device=dev)
    limit = rf"\({_native.PDB_ERR_LIMIT}\).*frames 129 > PDB_MAX_FRAMES"
    for mode in ("auto", "fp32", "tf32"):
        with engine(ctx, mode):
            with pytest.raises(_native.NativeError, match=limit):
                den(xb, t, zb)
            with pytest.raises(_native.NativeError, match=limit):
                ctx.p_sample(xb, 50, zb, draws[1])
            with pytest.raises(_native.NativeError, match=limit):
                ctx.sample_loop(zb, draws, None, None, 0)
    assert torch.equal(forward(den, dev, x, 50, z), before)
