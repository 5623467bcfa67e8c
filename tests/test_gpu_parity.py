"""GPU parity tests: the sm_90a path (through the C-ABI library) vs the reference fixtures
(tests/golden, produced by the reference's own modules) and vs the CPU oracle on seeded inputs.

Tolerances (fp32 end to end; the reference is fp32 too):
  * denoiser output eps:        |d| <= 3e-5 absolute (values are O(0.1..1); different summation order only)
  * one DDPM step (teacher-forced): 1e-5 relative to max |x|
  * Sampson gradient:           2e-4 of max |grad| vs the reference's fp32 autograd, 1e-4 vs the fp64 closed form
  * valid-match counts / pair-segment indexing / iteration counts / early exits: exact
  * GGS pose after a five-phase call: 2e-5 of max |pose| (the update is norm-clipped: 1e-4 |pose| per iteration)
"""
from functools import partial

import numpy as np
import pytest
import torch

from conftest import load_golden, matches_from
from oracle import pose_oracle as po
from oracle import sampson_f64 as s64

import posediffusion_b200 as pdb
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
FLAGS = ((1, 1, 1), (0, 0, 1), (1, 0, 0), (0, 1, 0))


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def golden_state():
    g = load_golden("denoiser.npz")
    return syn.random_denoiser_state(int(g["weight_seed"]), float(g["bias_std"]))


@pytest.fixture(scope="module")
def sampler(dev, golden_state):
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(golden_state, strict=True)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    return dif.to(dev)


@pytest.fixture(scope="module")
def ctx(sampler):
    return sampler.model.native_context()


def nan_close(actual, desired, atol):
    actual, desired = np.asarray(actual, dtype=np.float64), np.asarray(desired, dtype=np.float64)
    assert np.array_equal(np.isnan(actual), np.isnan(desired))
    ok = ~np.isnan(desired)
    np.testing.assert_allclose(actual[ok], desired[ok], rtol=0, atol=atol)


# ---------------------------------------------------------------------------------------------------
# denoiser / sampler
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["b1n5", "b1n20", "b2n20", "b1n80"])
def test_denoiser_forward_vs_reference(sampler, dev, tag):
    g = load_golden("denoiser.npz")
    x, z = torch.from_numpy(g[f"{tag}_x"]).to(dev), torch.from_numpy(g[f"{tag}_z"]).to(dev)
    t = torch.full((x.shape[0],), int(g[f"{tag}_t"]), dtype=torch.long, device=dev)
    eps = sampler.model(x, t, z).cpu().numpy()
    np.testing.assert_allclose(eps, g[f"{tag}_eps"], rtol=0, atol=3e-5)


@pytest.mark.parametrize("t", [99, 50, 11, 10, 9, 0])
def test_p_sample_teacher_forced_vs_reference(ctx, dev, t):
    g = load_golden("p_sample.npz")
    x, noise, z = (torch.from_numpy(g[k]).to(dev) for k in (f"t{t}_x", f"t{t}_noise", "z"))
    pred, mean, x0 = ctx.p_sample(x, t, z, None if t == 0 else noise)
    scale = np.abs(g[f"t{t}_x0"]).max()
    np.testing.assert_allclose(x0.cpu().numpy(), g[f"t{t}_x0"], rtol=0, atol=1e-5 * scale + 3e-5 * abs(float(po.diffusion_schedule()["sqrt_recipm1_alphas_cumprod"][t])))
    np.testing.assert_allclose(pred.cpu().numpy(), g[f"t{t}_pred"], rtol=0, atol=2e-5 * np.abs(g[f"t{t}_pred"]).max() + 1e-5)


def _self_consistent(sampler, z, draws, trail, steps, cond=None, start=0):
    """The fused loop must equal its own single-step API applied to its own trajectory (no chaos involved)."""
    ctx = sampler.model.native_context()
    for t in steps:
        k = 99 - t
        if cond is not None and t < start:
            got, _ = sampler.p_sample(trail[k].clone(), t, z, cond_fn=cond, cond_start_step=start)
            tol = 2e-5
        else:
            got, _, _ = ctx.p_sample(trail[k].contiguous(), t, z, None if t == 0 else draws[1 + k].contiguous())
            tol = 1e-6
        scale = trail[k + 1].abs().max().item()
        assert (got - trail[k + 1]).abs().max().item() <= tol * scale + 1e-7, t


def test_loop_ggs_off_vs_reference(sampler, dev):
    g = load_golden("loop.npz")
    z, draws = torch.from_numpy(g["z"]).to(dev), torch.from_numpy(g["draws"]).to(dev)
    pose, trail = sampler.p_sample_loop([1, 5, 9], z, None, 0, draws=draws)
    ref = g["off_trail"]
    assert trail.shape == ref.shape and torch.equal(pose, trail[-1]) and torch.equal(trail[0], draws[0])
    _self_consistent(sampler, z, draws, trail, range(99, -1, -1))
    # vs the reference: every step teacher-forced on the reference trajectory ...
    ctx = sampler.model.native_context()
    for t in range(99, -1, -1):
        k = 99 - t
        pred, _, _ = ctx.p_sample(torch.from_numpy(ref[k]).to(dev), t, z, None if t == 0 else draws[1 + k].contiguous())
        np.testing.assert_allclose(pred.cpu().numpy(), ref[k + 1], rtol=0, atol=3e-5 * np.abs(ref[k + 1]).max() + 1e-5)
    # ... and free-running while the (random-weight) dynamics have not yet amplified rounding differences
    # (the reference differs from itself by 6.6e-2 over 100 steps between 1 and 8 CPU threads, BASELINE.md §2)
    np.testing.assert_allclose(trail[:11].cpu().numpy(), ref[:11], rtol=0, atol=2e-3 * np.abs(ref[:11]).max())


def test_loop_ggs_on_vs_reference(sampler, dev):
    g = load_golden("loop.npz")
    m = matches_from(g, "on")
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=int(g["on_iter_num"]), min_matches=0, verbose=False)
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    z, draws = torch.from_numpy(g["z"]).to(dev), torch.from_numpy(g["draws"])
    slots = torch.cat([draws[:91], torch.zeros(10, *draws.shape[1:])]).to(dev)  # guided steps draw nothing
    pose, trail = sampler.p_sample_loop([1, 5, 9], z, cond, 10, draws=slots)
    ref = g["on_trail"]
    assert torch.isfinite(trail).all() and torch.equal(pose, trail[-1])
    _self_consistent(sampler, z, slots, trail, range(99, -1, -1), cond, 10)
    # guided steps teacher-forced on the reference trajectory through the public step API (p_sample + cond_fn)
    for t in range(9, -1, -1):
        got, _ = sampler.p_sample(torch.from_numpy(ref[99 - t]).to(dev), t, z, cond_fn=cond, cond_start_step=10)
        # this fixture is deliberately degenerate (random-weight trajectory vs unrelated matches: a handful of
        # borderline-valid matches carry the whole gradient), so one validity flip moves a focal entry by ~1e-4 |pose|
        np.testing.assert_allclose(got.cpu().numpy(), ref[100 - t], rtol=0, atol=2e-4 * np.abs(ref[100 - t]).max())
    # the fused loop and the generic-callable loop agree on the unguided prefix exactly and stay close afterwards
    generic = lambda mean, t: pdb.geometry_guided_sampling(mean, t, m, cfg)
    pose2, trail2 = sampler.p_sample_loop([1, 5, 9], z, generic, 10, draws=slots)
    assert (trail2[:91] - trail[:91]).abs().max().item() <= 1e-6 * trail[:91].abs().max().item()
    np.testing.assert_allclose(trail2[91].cpu().numpy(), trail[91].cpu().numpy(), rtol=0, atol=5e-5 * trail[91].abs().max().item())


def test_rng_draw_order_matches_reference(sampler, dev):
    """1 + 99 draws unguided, 1 + 90 with start_step 10, consumed in loop order on the device generator."""
    torch.manual_seed(123)
    d = sampler.draw_noise((1, 5, 9), dev, 10)
    torch.manual_seed(123)
    first = torch.randn(1, 5, 9, device=dev)
    rest = [torch.randn(1, 5, 9, device=dev) for _ in range(90)]
    assert torch.equal(d[0], first) and all(torch.equal(d[1 + k], rest[k]) for k in range(90))
    assert float(d[91:].abs().sum()) == 0.0


# ---------------------------------------------------------------------------------------------------
# Sampson error + gradient
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["scene6", "ragged5", "uniform5", "empty5", "diag4", "clamp4"])
@pytest.mark.parametrize("flags", FLAGS)
def test_sampson_eval_vs_reference(ctx, dev, tag, flags):
    g = load_golden("sampson.npz")
    m = matches_from(g, tag)
    key = f"{tag}_f{''.join(map(str, flags))}"
    pm = ctx.pack_matches(m)
    grad, sc, Fd, Gd = ctx.sampson_eval(pm, torch.from_numpy(g[f"{tag}_pose"]).to(dev), *map(bool, flags), dump=True)
    grad, sc = grad.cpu().numpy(), sc.cpu().numpy()
    n_ref = int(g[f"{key}_n_valid"])
    assert int(sc[1]) == n_ref
    nan_close(sc[2], g[f"{key}_logged"], 1e-5 * 10)
    c = s64.sampson_closed_form_f64(g[f"{tag}_pose"], m, *map(bool, flags))
    # per-segment F' and G against the closed form (segments are runs of equal pairs, in input order)
    i12 = m["i12"]
    runs = [0] + [i for i in range(1, len(i12)) if (i12[i] != i12[i - 1]).any()]
    assert pm.segments == len(runs)
    frames = m["img_shape"][0]
    Fd, Gd = Fd.cpu().numpy(), Gd.cpu().numpy()
    seen = {}
    for s, r in enumerate(runs):
        pid = int(i12[r, 0] * frames + i12[r, 1])
        Fref = c["F"][pid].reshape(-1)
        np.testing.assert_allclose(Fd[s], Fref, rtol=0, atol=2e-5 * max(np.abs(Fref).max(), 1e-30))
        seen.setdefault(pid, np.zeros(9))
        seen[pid] += Gd[s]
    for pid, Gsum in seen.items():
        Gref = c["G"][pid].reshape(-1)
        # G is an ill-conditioned intermediate (entries ~1e8 that largely cancel in the pose gradient): loose check here,
        # the pose gradient below is the quantity held to the stated tolerance
        nan_close(Gsum, Gref, 3e-3 * max(np.nanmax(np.abs(Gref)), 1e-30) if not np.all(np.isnan(Gref)) else 0)
    if n_ref == 0:
        return
    ref = g[f"{key}_grad"]
    gmax = np.nanmax(np.abs(ref))
    np.testing.assert_allclose(sc[0], g[f"{key}_loss"], rtol=2e-5)
    nan_close(grad, ref, 2e-4 * gmax)
    nan_close(grad, c["grad"], 1e-4 * gmax)
    assert np.array_equal(grad == 0, ref == 0)


@pytest.mark.parametrize("frames,per_pair,ragged", [(20, 256, False), (12, 100, True), (3, 5000, False), (40, 37, False)])
def test_sampson_eval_vs_oracle_seeded(ctx, dev, frames, per_pair, ragged):
    """Sizes the fixtures do not hold: many CTAs per problem, multi-chunk segment spans, ragged pairs."""
    m, gt, start = syn.scene_matches(frames, per_pair, seed=frames, ragged=ragged)
    pm = ctx.pack_matches(m)
    assert pm.m_total == len(m["kp1"])
    grad, sc, _, _ = ctx.sampson_eval(pm, torch.from_numpy(start).to(dev))
    prep = po.prepare_matches(m)
    pose = torch.from_numpy(start)[None].clone().requires_grad_(True)
    with torch.enable_grad():
        valid, logged = po.sampson_terms(pose, prep)
        valid.mean().backward()
    c = s64.sampson_closed_form_f64(start, m)
    assert abs(int(sc[1].item()) - len(valid)) <= 2 and abs(int(sc[1].item()) - c["n_valid"]) <= 2
    gmax = np.abs(c["grad"]).max()
    np.testing.assert_allclose(grad.cpu().numpy(), c["grad"], rtol=0, atol=3e-4 * gmax)
    # the reference's own fp32 chain (batched inverse, bmm) is the less accurate of the two: fp64 arbitrates
    np.testing.assert_allclose(grad.cpu().numpy(), pose.grad[0].numpy(), rtol=0, atol=1e-2 * gmax)
    np.testing.assert_allclose(sc[2].item(), float(logged), rtol=1e-4)


def test_sampson_properties_at_full_size(ctx, dev):
    """BASELINE config 3 size (N=20, 380 ordered pairs x 2048 = 778 240 matches): size-independent properties."""
    frames, per_pair = 20, 2048
    m, gt, start = syn.scene_matches(frames, per_pair, seed=77)
    pose = torch.from_numpy(start).to(dev)
    pm = ctx.pack_matches(m)
    assert (pm.m_total, pm.segments, pm.rounds) == (380 * 2048, 380, 380 * 64)
    g1, s1, _, _ = ctx.sampson_eval(pm, pose)
    # (a) run-to-run: identical counts, gradient equal up to atomics ordering
    g2, s2, _, _ = ctx.sampson_eval(pm, pose)
    assert s1[1].item() == s2[1].item()
    gmax = g1.abs().max().item()
    assert (g1 - g2).abs().max().item() <= 2e-5 * gmax
    # (b) permuting the pair order leaves the mean gradient unchanged
    order = np.random.default_rng(0).permutation(380)
    idx = (order[:, None] * per_pair + np.arange(per_pair)[None]).reshape(-1)
    mp = {"kp1": m["kp1"][idx], "kp2": m["kp2"][idx], "i12": m["i12"][idx], "img_shape": m["img_shape"]}
    g3, s3, _, _ = ctx.sampson_eval(ctx.pack_matches(mp), pose)
    assert s3[1].item() == s1[1].item()
    assert (g1 - g3).abs().max().item() <= 5e-5 * gmax
    # (c) duplicating every match leaves mean loss / gradient unchanged and doubles the valid count
    md = {k: (np.concatenate([v, v]) if k != "img_shape" else v) for k, v in m.items()}
    g4, s4, _, _ = ctx.sampson_eval(ctx.pack_matches(md), pose)
    assert s4[1].item() == 2 * s1[1].item()
    assert (g1 - g4).abs().max().item() <= 5e-5 * gmax and abs(s4[0].item() - s1[0].item()) <= 1e-4 * s1[0].item()
    # (d) detached blocks: flags partition the full gradient exactly
    gR, _, _, _ = ctx.sampson_eval(pm, pose, True, False, False)
    gT, _, _, _ = ctx.sampson_eval(pm, pose, False, True, False)
    gF, _, _, _ = ctx.sampson_eval(pm, pose, False, False, True)
    assert (gR[:, :3] == 0).all() and (gR[:, 7:] == 0).all() and (gT[:, 3:] == 0).all() and (gF[:, :7] == 0).all()
    assert ((gR + gT + gF) - g1).abs().max().item() <= 5e-5 * gmax
    # (e) noise-free correspondences have (near) zero error at the ground-truth pose
    m0, gt0, _ = syn.scene_matches(frames, 256, seed=78, pixel_noise=0.0)
    _, s0, _, _ = ctx.sampson_eval(ctx.pack_matches(m0), torch.from_numpy(gt0).to(dev))
    assert s0[1].item() == 380 * 256 and s0[0].item() < 1e-4


@pytest.mark.parametrize("mode", ["resident", "stream"])
def test_streaming_paths_agree(ctx, dev, mode, monkeypatch):
    """The three ways stage 1 reads matches (shared-memory resident slice, bulk-async ring, plain global loads for
    CTAs that own more than 128 pair segments) must give the same statistics and gradient."""
    if mode == "stream":
        monkeypatch.setenv("PDB_GGS_FORCE_STREAM", "1")
    else:
        monkeypatch.delenv("PDB_GGS_FORCE_STREAM", raising=False)
    # (a) config-3-like shape
    m, gt, start = syn.scene_matches(12, 300, seed=91, ragged=True)
    pose = torch.from_numpy(start).to(dev)
    grad, sc, _, _ = ctx.sampson_eval(ctx.pack_matches(m), pose)
    c = s64.sampson_closed_form_f64(start, m)
    assert abs(int(sc[1].item()) - c["n_valid"]) <= 2
    np.testing.assert_allclose(grad.cpu().numpy(), c["grad"], rtol=0, atol=3e-4 * np.abs(c["grad"]).max())
    # (b) pathological input: two pairs alternating row by row -> every match is its own segment (> 128 per CTA)
    frames, rows = 4, 40000
    rng = np.random.default_rng(5)
    mm, _, st4 = syn.scene_matches(frames, rows // 12 + 1, seed=92)
    pick = np.where((mm["i12"][:, 0] == 0) & (mm["i12"][:, 1] == 1))[0]
    pick2 = np.where((mm["i12"][:, 0] == 2) & (mm["i12"][:, 1] == 3))[0]
    n = min(len(pick), len(pick2))
    order = np.stack([pick[:n], pick2[:n]], 1).reshape(-1)
    inter = {"kp1": mm["kp1"][order], "kp2": mm["kp2"][order], "i12": mm["i12"][order], "img_shape": mm["img_shape"]}
    pm = ctx.pack_matches(inter)
    assert pm.segments == 2 * n
    grad, sc, _, _ = ctx.sampson_eval(pm, torch.from_numpy(st4).to(dev))
    c = s64.sampson_closed_form_f64(st4, inter)
    assert abs(int(sc[1].item()) - c["n_valid"]) <= 2
    np.testing.assert_allclose(grad.cpu().numpy(), c["grad"], rtol=0, atol=3e-4 * np.abs(c["grad"]).max())
    # (c) a short five-phase run agrees between the modes through the oracle
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = 6
    p0 = torch.from_numpy(start)[None].to(dev).clone()
    ctx.ggs([ctx.pack_matches(m)], p0, cfg, want_stats=False)
    want = po.geometry_guided_sampling(torch.from_numpy(start)[None], 5, m, cfg)
    np.testing.assert_allclose(p0[0].cpu().numpy(), want[0].numpy(), rtol=0, atol=3e-5 * np.abs(want).max().item())


def test_streaming_ring_at_config5_size(ctx, dev):
    """BASELINE config 5 size (N=80, 6320 ordered pairs x 4096 = 25 886 720 matches, 414 MB): the bulk-async ring streams
    ~340 rounds per warp.  Size-independent checks: statistics are additive over a split of the pairs, the valid count is
    reproducible, and the gradient of the union is the count-weighted mean of the parts."""
    frames, per_pair = 80, 4096
    m = syn.uniform_matches(frames, per_pair, seed=3)
    _, _, start = syn.scene_matches(frames, 2, seed=4)
    pose = torch.from_numpy(start).to(dev)
    pm = ctx.pack_matches(m)
    assert (pm.m_total, pm.segments, pm.rounds) == (6320 * 4096, 6320, 6320 * 128)
    g_all, s_all, _, _ = ctx.sampson_eval(pm, pose)
    g_again, s_again, _, _ = ctx.sampson_eval(pm, pose)
    assert s_all[1].item() == s_again[1].item() and s_all[1].item() > 1000
    half = (6320 // 2) * per_pair
    parts = []
    for lo, hi in ((0, half), (half, 6320 * per_pair)):
        sub = {"kp1": m["kp1"][lo:hi], "kp2": m["kp2"][lo:hi], "i12": m["i12"][lo:hi], "img_shape": m["img_shape"]}
        g, sc, _, _ = ctx.sampson_eval(ctx.pack_matches(sub), pose)
        parts.append((g, sc))
    n1, n2 = parts[0][1][1].item(), parts[1][1][1].item()
    assert n1 + n2 == s_all[1].item()
    loss = (parts[0][1][0].item() * n1 + parts[1][1][0].item() * n2) / (n1 + n2)
    assert abs(loss - s_all[0].item()) <= 2e-4 * abs(s_all[0].item())
    g_mix = (parts[0][0] * n1 + parts[1][0] * n2) / (n1 + n2)
    assert (g_mix - g_all).abs().max().item() <= 2e-4 * g_all.abs().max().item()
    assert (g_all - g_again).abs().max().item() <= 5e-5 * g_all.abs().max().item()


def test_matches_pack_validation(ctx):
    m = syn.uniform_matches(4, 8, seed=1)
    bad = dict(m)
    bad["i12"] = m["i12"].copy()
    bad["i12"][5, 1] = 4
    with pytest.raises(ValueError):
        ctx.pack_matches(bad)
    empty = {"kp1": np.zeros((0, 2)), "kp2": np.zeros((0, 2)), "i12": np.zeros((0, 2), np.int64), "img_shape": (4, 3, 224, 224)}
    pm = ctx.pack_matches(empty)
    assert (pm.m_total, pm.segments, pm.rounds) == (0, 0, 0)


# ---------------------------------------------------------------------------------------------------
# geometry-guided sampling
# ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["scene5", "scene8"])
def test_ggs_five_phases_vs_reference(ctx, dev, tag):
    g = load_golden("ggs.npz")
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = int(g["iter_num"])
    m = matches_from(g, tag)
    pose = torch.from_numpy(g[f"{tag}_pose"])[None].to(dev).clone()
    stats = ctx.ggs([ctx.pack_matches(m)], pose, cfg)
    row = _native.stats_to_numpy(stats)[0]
    ref = g[f"{tag}_out"]
    np.testing.assert_allclose(pose[0].cpu().numpy(), ref, rtol=0, atol=2e-5 * np.abs(ref).max())
    n = cfg["iter_num"]
    assert list(row["iters"]) == [2 * n, n, n, n, 2 * n] and int(row["dropped"].sum()) == int(g[f"{tag}_drops"])
    np.testing.assert_allclose(row["sampson"], g[f"{tag}_log"], rtol=2e-3)


def test_ggs_early_exit_vs_reference(ctx, dev, capsys):
    g = load_golden("ggs.npz")
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = int(g["iter_num"])
    m = matches_from(g, "drop")
    pose = torch.from_numpy(g["drop_pose"])[None].to(dev).clone()
    out = pdb.geometry_guided_sampling(pose, 3, m, cfg)  # the public drop-in, printing like the reference
    text = capsys.readouterr().out
    assert text.count("Drop this pair because of insufficient valid matches") == int(g["drop_drops"]) == 5
    assert text.count("t=03 | sampson=") == 5
    assert np.array_equal(out[0].cpu().numpy(), g["drop_out"])  # no update at all


def test_ggs_long_run_vs_oracle(ctx, dev):
    """Default iteration counts (700 inner iterations) on a consistent scene: agreement with the CPU oracle and descent."""
    m, gt, start = syn.scene_matches(6, 128, seed=5)
    cfg = syn.default_ggs_cfg()
    pose = torch.from_numpy(start)[None].to(dev).clone()
    pm = ctx.pack_matches(m)
    _, sc0, _, _ = ctx.sampson_eval(pm, pose[0].contiguous())
    stats = _native.stats_to_numpy(ctx.ggs([pm], pose, cfg))[0]
    log = []
    want = po.geometry_guided_sampling(torch.from_numpy(start)[None], 5, m, cfg, log=log)
    assert list(stats["iters"]) == [e["iters"] for e in log] == [200, 100, 100, 100, 200]
    np.testing.assert_allclose(pose[0].cpu().numpy(), want[0].numpy(), rtol=0, atol=1e-3 * np.abs(want).max().item())
    np.testing.assert_allclose(stats["sampson"], [e["sampson"] for e in log], rtol=2e-2)
    assert stats["sampson"][-1] < sc0[2].item()  # the optimisation lowered the (clamped) mean Sampson error


def test_ggs_batch_equals_singles(ctx, dev):
    """B independent sequences in one launch == B single launches (the path shards over sequences)."""
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = 5
    sets = [syn.scene_matches(7, 64 + 16 * s, seed=40 + s) for s in range(3)]
    packs = [ctx.pack_matches(s[0]) for s in sets]
    starts = torch.stack([torch.from_numpy(s[2]) for s in sets]).to(dev)
    batch = starts.clone()
    ctx.ggs(packs, batch, cfg)
    for i in range(3):
        single = starts[i : i + 1].clone()
        ctx.ggs([packs[i]], single, cfg)
        np.testing.assert_allclose(batch[i].cpu().numpy(), single[0].cpu().numpy(), rtol=0, atol=1e-5 * single.abs().max().item())


def test_batched_denoiser_equals_singles(sampler, dev):
    x = torch.randn(3, 20, 9, device=dev)
    z = torch.randn(3, 20, 384, device=dev)
    t = torch.full((3,), 42, dtype=torch.long, device=dev)
    full = sampler.model(x, t, z)
    for i in range(3):
        one = sampler.model(x[i : i + 1].contiguous(), t[:1], z[i : i + 1].contiguous())
        np.testing.assert_allclose(full[i].cpu().numpy(), one[0].cpu().numpy(), rtol=0, atol=1e-6)


def test_host_buffer_entry_equals_device_entry(sampler, dev):
    """pdb_sample_loop_host (pinned host buffers, the e2e call) == pdb_sample_loop on device buffers."""
    ctx = sampler.model.native_context()
    frames = 6
    m, _, _ = syn.scene_matches(frames, 48, seed=61)
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=3, min_matches=0, verbose=False)
    z = syn.random_features(2, frames, 61)
    draws = syn.predraw_noise(2, frames, seed=61)
    packs = [ctx.pack_matches(m), ctx.pack_matches(m)]
    pose_d, trail_d, stats_d = ctx.sample_loop(z.to(dev), draws.to(dev), packs, cfg, 10)
    pose_h = np.zeros((2, frames, 9), np.float32)
    trail_h = np.zeros((101, 2, frames, 9), np.float32)
    stats_h = np.zeros(10 * 2, dtype=_native.GGS_STATS_DTYPE)
    ctx.sample_loop_host(z.numpy(), draws.numpy(), packs, cfg, 10, pose_h, trail_h, stats_h)
    scale = np.abs(trail_h).max()
    # identical kernels on identical data; only the GGS atomics' ordering may differ between the two runs
    np.testing.assert_allclose(trail_h[:91], trail_d[:91].cpu().numpy(), rtol=0, atol=0)
    np.testing.assert_allclose(pose_h, pose_d.cpu().numpy(), rtol=0, atol=1e-3 * scale)
    dev_stats = _native.stats_to_numpy(stats_d)
    assert np.array_equal(stats_h["iters"], dev_stats["iters"]) and stats_h["iters"].sum() == 10 * 2 * 21
    # both sequences of the batch saw the same inputs except z / noise
    assert not np.allclose(pose_h[0], pose_h[1])


@pytest.mark.parametrize("B,N", [(1, 20), (2, 20), (1, 5), (3, 13), (1, 80)])
def test_denoiser_handover_modes_bit_identical(sampler, dev, B, N):
    """The two stage hand-overs of the persistent denoiser kernel (group barriers = default, flag-carrying activation words)
    run the same arithmetic in the same order: the whole unguided trajectory (100 steps, one launch) is bit-identical.
    Run twice in the flagged mode: the second launch reuses buffers that hold the first launch's (older-version) words."""
    ctx = sampler.model.native_context()
    z = syn.random_features(B, N, 5).to(dev)
    draws = syn.predraw_noise(B, N, seed=5).to(dev)
    try:
        ctx.set_denoiser_engine("fp32")
        ctx.set_denoiser_handover(False)
        pose_a, trail_a, _ = ctx.sample_loop(z, draws, None, None, 0)
        ctx.set_denoiser_handover(True)
        pose_b, trail_b, _ = ctx.sample_loop(z, draws, None, None, 0)
        pose_c, trail_c, _ = ctx.sample_loop(z, draws, None, None, 0)
    finally:
        ctx.set_denoiser_handover(False)
        ctx.set_denoiser_engine("auto")
    assert torch.isfinite(trail_a).all()
    assert torch.equal(trail_a, trail_b) and torch.equal(pose_a, pose_b)
    assert torch.equal(trail_a, trail_c) and torch.equal(pose_a, pose_c)


def test_host_matches_entry_equals_pack_then_host_entry(sampler, dev):
    """pdb_sample_loop_host_matches (reference-format matches in, packing overlapped with the unguided steps) ==
    pdb_matches_pack + pdb_sample_loop_host; bad input is rejected and leaves the context usable."""
    ctx = sampler.model.native_context()
    frames = 6
    sets = [syn.scene_matches(frames, 48 + 16 * s, seed=71 + s)[0] for s in range(2)]
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=3, min_matches=0, verbose=False)
    z = syn.random_features(2, frames, 71).numpy()
    draws = syn.predraw_noise(2, frames, seed=71).numpy()
    for start in (10, 0, 100):  # usual split; guidance never starts; no unguided prefix at all
        packs = [ctx.pack_matches(m) for m in sets]
        want, want_trail = np.zeros((2, frames, 9), np.float32), np.zeros((101, 2, frames, 9), np.float32)
        want_stats = np.zeros(max(start, 1) * 2, dtype=_native.GGS_STATS_DTYPE)
        ctx.sample_loop_host(z, draws, packs, cfg, start, want, want_trail, want_stats)
        got, got_trail = np.zeros_like(want), np.zeros_like(want_trail)
        got_stats = np.zeros_like(want_stats)
        ctx.sample_loop_host_matches(z, draws, sets, cfg, start, got, got_trail, got_stats)
        np.testing.assert_array_equal(got_trail[: 101 - start], want_trail[: 101 - start])  # unguided part: no atomics
        if start == 100:
            # guidance on pure noise with random weights diverges (both runs; the summation order of the exchange differs between
            # two launches and the divergence amplifies it): only the bookkeeping is comparable
            assert (got_stats["iters"] > 0).all() and (want_stats["iters"] > 0).all()  # all 100 x 2 guided steps ran
            continue
        scale = np.abs(want_trail).max()
        np.testing.assert_allclose(got, want, rtol=0, atol=1e-3 * scale)
        assert np.array_equal(got_stats["iters"], want_stats["iters"])
    bad = dict(sets[0])
    bad["i12"] = np.array(bad["i12"]).copy()
    bad["i12"][3, 1] = frames
    with pytest.raises(ValueError, match="outside"):
        ctx.sample_loop_host_matches(z, draws, [sets[0], bad], cfg, 10, got)
    with pytest.raises(ValueError, match="one per sequence"):
        ctx.sample_loop_host_matches(z, draws, sets[:1], cfg, 10, got)
    ctx.sample_loop_host_matches(z, draws, sets, cfg, 10, got)  # still usable
    assert np.isfinite(got).all()


def test_pose_diffusion_model_api(dev, golden_state):
    model = pdb.PoseDiffusionModel(
        pose_encoding_type="absT_quaR_logFL", IMAGE_FEATURE_EXTRACTOR=None,
        DIFFUSER={"_target_": "models.GaussianDiffusion", "beta_schedule": "custom"},
        DENOISER={"_target_": "models.Denoiser", "TRANSFORMER": dict(TRANSFORMER, _target_="models.TransformerEncoderWrapper")},
    ).to(dev)
    model.diffuser.model.load_state_dict(golden_state, strict=True)
    z = torch.randn(1, 6, 384, device=dev)
    torch.manual_seed(0)
    out = model(z=z, training=False)
    cams = out["pred_cameras"]
    assert len(cams) == 6 and torch.isfinite(cams.R).all() and torch.isfinite(cams.T).all()
    torch.manual_seed(0)
    again = model(z=z, training=False)["pred_cameras"]
    assert torch.equal(cams.T, again.T)  # deterministic given the seed (GGS off: no atomics on the path)


def test_example_demo_runs(capsys):
    import importlib.util, os
    from conftest import ROOT

    spec = importlib.util.spec_from_file_location("demo_synthetic", os.path.join(ROOT, "examples", "demo_synthetic.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.main(frames=6, matches_per_pair=64)
    out = capsys.readouterr().out
    assert "GGS off" in out and "GGS on" in out


def test_colmap_ingestion_equals_reference_format_ingestion(ctx, dev):
    """pdb_matches_pack_colmap (remap fused into the gather) == pdb_matches_pack of the reference function's output."""
    from oracle.make_golden import synthetic_colmap_tables
    from posediffusion_b200.match_extraction import pack_colmap_matches

    g = load_golden("colmap.npz")
    matches, keypoints, image_info = synthetic_colmap_tables()
    img_shape = (5, 3, 224, 224)
    ref_dict = {"kp1": g["kp1"], "kp2": g["kp2"], "i12": g["i12"], "img_shape": img_shape}
    pm_ref = ctx.pack_matches(ref_dict)
    pm_col = pack_colmap_matches(ctx, matches, keypoints, image_info, img_shape)
    assert (pm_col.m_total, pm_col.segments, pm_col.rounds) == (pm_ref.m_total, pm_ref.segments, pm_ref.rounds)
    pose = torch.from_numpy(syn.scene_matches(5, 4, seed=1)[2]).to(dev)
    for smax in (10.0, 1e9):  # with a huge threshold every match is valid: the sums see every coordinate
        g1, s1, F1, G1 = ctx.sampson_eval(pm_ref, pose, sampson_max=smax, dump=True)
        g2, s2, F2, G2 = ctx.sampson_eval(pm_col, pose, sampson_max=smax, dump=True)
        assert s1[1].item() == s2[1].item()
        assert torch.equal(F1, F2)
        scale = G1.abs().max().item()
        assert (G1 - G2).abs().max().item() <= 1e-4 * scale
    bad = dict(matches)
    bad[(1, 2)] = np.array([[0, 10_000]])
    with pytest.raises(ValueError):
        pack_colmap_matches(ctx, bad, keypoints, image_info, img_shape)


def test_cond_start_step_edges(sampler, dev):
    """cond_start_step = 0 -> the guidance callable is never used (gaussian_diffuser.py:270: t < 0 is never true);
    a start step of 3 guides exactly t = 2, 1, 0 and consumes 1 + 97 draws."""
    frames = 5
    m, _, _ = syn.scene_matches(frames, 40, seed=71)
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=2, min_matches=0, verbose=False)
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    z = syn.random_features(1, frames, 71).to(dev)
    draws = syn.predraw_noise(1, frames, seed=71).to(dev)
    p_off, t_off = sampler.p_sample_loop([1, frames, 9], z, None, 0, draws=draws)
    p_zero, t_zero = sampler.p_sample_loop([1, frames, 9], z, cond, 0, draws=draws)
    assert torch.equal(t_off, t_zero)
    p3, t3 = sampler.p_sample_loop([1, frames, 9], z, cond, 3, draws=draws)
    assert torch.equal(t3[:98], t_off[:98]) and not torch.equal(t3[98], t_off[98])
    stats = _native.stats_to_numpy(sampler.last_ggs_stats).reshape(3, 1)
    assert (stats["iters"] == np.array([4, 2, 2, 2, 4])).all()
    torch.manual_seed(7)
    d3 = sampler.draw_noise((1, frames, 9), dev, 3)
    assert float(d3[98:].abs().sum()) == 0.0 and float(d3[97].abs().sum()) > 0.0


def test_two_devices_in_one_process():
    """One pdb_context per GPU inside a single process (the normal deployment is one process per GPU)."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    m, _, start = syn.scene_matches(6, 50, seed=81)
    ref = s64.sampson_closed_form_f64(start, m)
    state = syn.random_denoiser_state(2)
    for index in (0, 1):
        d = torch.device("cuda", index)
        c = _native.Context.get(d)
        grad, sc, _, _ = c.sampson_eval(c.pack_matches(m), torch.from_numpy(start).to(d))
        assert int(sc[1].item()) == ref["n_valid"]
        np.testing.assert_allclose(grad.cpu().numpy(), ref["grad"], rtol=0, atol=3e-4 * np.abs(ref["grad"]).max())
        den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
        den.load_state_dict(state, strict=True)
        den = den.to(d)
        eps = den(torch.zeros(1, 6, 9, device=d), torch.zeros(1, dtype=torch.long, device=d), torch.ones(1, 6, 384, device=d))
        assert torch.isfinite(eps).all()
        if index == 0:
            first = eps.cpu()
        else:
            assert torch.allclose(first, eps.cpu(), atol=1e-6)


def test_fused_loop_rejects_wrong_problem_count_and_frame_count(sampler, dev):
    """ADVICE r1: B > 1 with a single matches_dict, or a dict whose img_shape[0] differs from the pose's frame count, must
    raise instead of indexing past the problem array / striding the pose with the wrong frame count."""
    ctx = sampler.model.native_context()
    frames = 6
    m, _, _ = syn.scene_matches(frames, 16, seed=3)
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=1, verbose=False)
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=cfg)
    z2 = syn.random_features(2, frames, 1).to(dev)
    with pytest.raises(ValueError, match="match sets for a batch"):
        sampler.p_sample_loop([2, frames, 9], z2, cond, 10)
    z7 = syn.random_features(1, frames + 1, 1).to(dev)
    with pytest.raises(ValueError, match="img_shape"):
        sampler.p_sample_loop([1, frames + 1, 9], z7, cond, 10)
    # the library itself refuses too (a caller that binds the C ABI directly)
    import ctypes as C
    pm = ctx.pack_matches(m)
    draws = syn.predraw_noise(2, frames, seed=1).to(dev)
    pose = torch.empty(2, frames, 9, device=dev)
    conf = _native.ggs_config_struct(cfg)
    arr = ctx._problem_array([pm])
    rc = ctx.lib.pdb_sample_loop(ctx.handle, z2.data_ptr(), draws.data_ptr(), 2, frames, arr, 1, C.byref(conf), 10, pose.data_ptr(),
                                 None, None, None)
    assert rc == _native.PDB_ERR_INVALID and b"match sets" in ctx.lib.pdb_last_error(ctx.handle)
    draws7 = syn.predraw_noise(1, frames + 1, seed=1).to(dev)
    rc = ctx.lib.pdb_sample_loop(ctx.handle, z7.data_ptr(), draws7.data_ptr(), 1, frames + 1, arr, 1, C.byref(conf), 10,
                                 pose.data_ptr(), None, None, None)
    assert rc == _native.PDB_ERR_INVALID and b"frames" in ctx.lib.pdb_last_error(ctx.handle)
