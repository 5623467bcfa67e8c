"""GPU parity tests of the paired match-stream layout (csrc/ggs_layout.cuh, `pdb_ggs_layout(ctx, 1)`).

Every kernel instantiation the library ships runs here on the device (`ggs_entry<*, true>` as well as `<*, false>`):
the same fixtures and tolerances as tests/test_gpu_parity.py; against the plain layout the statistics must agree exactly
(valid counts) or up to summation order (sums).
"""
import os

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
FLAGS = ((1, 1, 1), (0, 0, 1), (1, 0, 0), (0, 1, 0))


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


def nan_close(actual, desired, atol):
    actual, desired = np.asarray(actual, dtype=np.float64), np.asarray(desired, dtype=np.float64)
    assert np.array_equal(np.isnan(actual), np.isnan(desired))
    ok = ~np.isnan(desired)
    np.testing.assert_allclose(actual[ok], desired[ok], rtol=0, atol=atol)


@pytest.mark.parametrize("tag", ["scene6", "ragged5", "uniform5", "empty5", "diag4", "clamp4"])
@pytest.mark.parametrize("flags", FLAGS)
def test_sampson_eval_paired_vs_reference_and_plain(ctx, dev, tag, flags):
    g = load_golden("sampson.npz")
    m = matches_from(g, tag)
    key = f"{tag}_f{''.join(map(str, flags))}"
    pose = torch.from_numpy(g[f"{tag}_pose"]).to(dev)
    pm1, pm0 = pack(ctx, m, "paired"), pack(ctx, m, "plain")
    assert pm1.segments == pm0.segments and pm1.rounds % 2 == 0 and pm1.rounds >= pm0.rounds
    grad, sc, Fd, Gd = ctx.sampson_eval(pm1, pose, *map(bool, flags), dump=True)
    grad0, sc0, Fd0, Gd0 = ctx.sampson_eval(pm0, pose, *map(bool, flags), dump=True)
    assert int(sc[1].item()) == int(sc0[1].item()) == int(g[f"{key}_n_valid"])
    assert torch.equal(Fd, Fd0)  # F' does not depend on the stream layout
    gs = Gd0.abs().max().item() + 1e-30
    nan_close((Gd / gs).cpu().numpy(), (Gd0 / gs).cpu().numpy(), 1e-5)
    nan_close(sc[2].item(), g[f"{key}_logged"], 1e-5 * 10)
    if int(sc[1].item()) == 0:
        return
    ref = g[f"{key}_grad"]
    gmax = np.nanmax(np.abs(ref))
    np.testing.assert_allclose(sc[0].item(), g[f"{key}_loss"], rtol=2e-5)
    nan_close(grad.cpu().numpy(), ref, 2e-4 * gmax)
    c = s64.sampson_closed_form_f64(g[f"{tag}_pose"], m, *map(bool, flags))
    nan_close(grad.cpu().numpy(), c["grad"], 1e-4 * gmax)
    assert np.array_equal(grad.cpu().numpy() == 0, ref == 0)


@pytest.mark.parametrize("frames,per_pair,ragged", [(20, 256, False), (12, 100, True), (3, 5000, False), (40, 37, False), (20, 2048, False)])
@pytest.mark.parametrize("force_stream", [False, True])
def test_sampson_eval_paired_seeded_sizes(ctx, dev, frames, per_pair, ragged, force_stream, monkeypatch):
    """Many CTAs per problem, ragged pairs, config-3 size; shared-memory resident walk and the bulk-async ring."""
    if force_stream:
        monkeypatch.setenv("PDB_GGS_FORCE_STREAM", "1")
    else:
        monkeypatch.delenv("PDB_GGS_FORCE_STREAM", raising=False)
    m, gt, start = syn.scene_matches(frames, per_pair, seed=frames, ragged=ragged)
    pose = torch.from_numpy(start).to(dev)
    g1, s1, _, _ = ctx.sampson_eval(pack(ctx, m, "paired"), pose)
    g0, s0, _, _ = ctx.sampson_eval(pack(ctx, m, "plain"), pose)
    assert s1[1].item() == s0[1].item()
    gmax = g0.abs().max().item()
    assert (g1 - g0).abs().max().item() <= 5e-5 * gmax
    np.testing.assert_allclose(s1[:3].cpu().numpy(), s0[:3].cpu().numpy(), rtol=2e-5)
    c = s64.sampson_closed_form_f64(start, m)
    assert abs(int(s1[1].item()) - c["n_valid"]) <= 2
    # fp32 is the limit at the config-3 size (778 240 matches): the reference's own fp32 operator sequence is 3.3e-4 * max|grad| away
    # from float64 there (tests/test_gpu_fullsize.py states the measurement)
    tol = 1e-3 if len(m["kp1"]) > 500000 else 3e-4
    np.testing.assert_allclose(g1.cpu().numpy(), c["grad"], rtol=0, atol=tol * np.abs(c["grad"]).max())


def test_paired_single_match_segments_and_register_stream_walk(ctx, dev, monkeypatch):
    """Two pairs alternating row by row: every match is its own segment (64-row units that hold one row), > 128 segments per
    CTA -> the register-stream walk."""
    monkeypatch.setenv("PDB_GGS_FORCE_STREAM", "1")
    mm, _, st4 = syn.scene_matches(4, 40000 // 12 + 1, seed=92)
    pick = np.where((mm["i12"][:, 0] == 0) & (mm["i12"][:, 1] == 1))[0]
    pick2 = np.where((mm["i12"][:, 0] == 2) & (mm["i12"][:, 1] == 3))[0]
    n = min(len(pick), len(pick2))
    order = np.stack([pick[:n], pick2[:n]], 1).reshape(-1)
    inter = {"kp1": mm["kp1"][order], "kp2": mm["kp2"][order], "i12": mm["i12"][order], "img_shape": mm["img_shape"]}
    pm = pack(ctx, inter, "paired")
    assert (pm.segments, pm.rounds) == (2 * n, 4 * n)
    grad, sc, _, _ = ctx.sampson_eval(pm, torch.from_numpy(st4).to(dev))
    c = s64.sampson_closed_form_f64(st4, inter)
    assert abs(int(sc[1].item()) - c["n_valid"]) <= 2
    np.testing.assert_allclose(grad.cpu().numpy(), c["grad"], rtol=0, atol=3e-4 * np.abs(c["grad"]).max())


def test_paired_ring_at_config5_size(ctx, dev):
    """BASELINE config 5 (414 MB per inner iteration through the bulk-async ring): paired == plain."""
    frames, per_pair = 80, 4096
    m = syn.uniform_matches(frames, per_pair, seed=3)
    _, _, start = syn.scene_matches(frames, 2, seed=4)
    pose = torch.from_numpy(start).to(dev)
    pm1 = pack(ctx, m, "paired")
    assert (pm1.m_total, pm1.segments, pm1.rounds) == (6320 * 4096, 6320, 6320 * 128)
    g1, s1, _, _ = ctx.sampson_eval(pm1, pose)
    del pm1
    g0, s0, _, _ = ctx.sampson_eval(pack(ctx, m, "plain"), pose)
    assert s1[1].item() == s0[1].item() and s1[1].item() > 1000
    assert (g1 - g0).abs().max().item() <= 5e-5 * g0.abs().max().item()
    assert abs(s1[0].item() - s0[0].item()) <= 2e-5 * abs(s0[0].item())


@pytest.mark.parametrize("tag", ["scene5", "scene8"])
def test_ggs_five_phases_paired_vs_reference(ctx, dev, tag):
    g = load_golden("ggs.npz")
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = int(g["iter_num"])
    m = matches_from(g, tag)
    pose = torch.from_numpy(g[f"{tag}_pose"])[None].to(dev).clone()
    row = _native.stats_to_numpy(ctx.ggs([pack(ctx, m, "paired")], pose, cfg))[0]
    ref = g[f"{tag}_out"]
    np.testing.assert_allclose(pose[0].cpu().numpy(), ref, rtol=0, atol=2e-5 * np.abs(ref).max())
    n = cfg["iter_num"]
    assert list(row["iters"]) == [2 * n, n, n, n, 2 * n] and int(row["dropped"].sum()) == int(g[f"{tag}_drops"])
    np.testing.assert_allclose(row["sampson"], g[f"{tag}_log"], rtol=2e-3)


def test_ggs_long_run_and_batches_paired(ctx, dev):
    cfg = syn.default_ggs_cfg()
    m, gt, start = syn.scene_matches(6, 128, seed=5)
    pose = torch.from_numpy(start)[None].to(dev).clone()
    stats = _native.stats_to_numpy(ctx.ggs([pack(ctx, m, "paired")], pose, cfg))[0]
    want = po.geometry_guided_sampling(torch.from_numpy(start)[None], 5, m, cfg)
    assert list(stats["iters"]) == [200, 100, 100, 100, 200]
    np.testing.assert_allclose(pose[0].cpu().numpy(), want[0].numpy(), rtol=0, atol=1e-3 * np.abs(want).max().item())
    # batch of three sequences in one launch == singles; a batch must not mix layouts
    cfg["iter_num"] = 5
    sets = [syn.scene_matches(7, 64 + 16 * s, seed=40 + s) for s in range(3)]
    packs = [pack(ctx, s[0], "paired") for s in sets]
    starts = torch.stack([torch.from_numpy(s[2]) for s in sets]).to(dev)
    batch = starts.clone()
    ctx.ggs(packs, batch, cfg)
    for i in range(3):
        single = starts[i : i + 1].clone()
        ctx.ggs([packs[i]], single, cfg)
        np.testing.assert_allclose(batch[i].cpu().numpy(), single[0].cpu().numpy(), rtol=0, atol=1e-5 * single.abs().max().item())
    with pytest.raises(_native.NativeError, match="same stream layout"):
        ctx.ggs([packs[0], pack(ctx, sets[1][0], "plain")], starts[:2].clone(), cfg)


def test_sample_loop_paired_equals_plain(dev):
    """Whole p_sample_loop with GGS on: the trajectory with paired match sets equals the plain one up to summation order."""
    state = syn.random_denoiser_state(3, 0.05)
    den = pdb.Denoiser(TRANSFORMER=dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1,
                                        batch_first=True, norm_first=True))
    den.load_state_dict(state, strict=True)
    den = den.to(dev)
    c = den.native_context()
    frames = 8
    m, _, _ = syn.scene_matches(frames, 200, seed=11)
    z = syn.random_features(1, frames, 2).to(dev)
    draws = syn.predraw_noise(1, frames, seed=2).to(dev)
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = 10
    out = {}
    for layout in ("plain", "paired"):
        pose, trail, _ = c.sample_loop(z, draws, [pack(c, m, layout)], cfg, cfg["start_step"])
        out[layout] = (pose.cpu().numpy(), trail.cpu().numpy())
    scale = np.abs(out["plain"][1]).max()
    np.testing.assert_allclose(out["paired"][1], out["plain"][1], rtol=0, atol=2e-3 * scale)  # atomics order + 10 chaotic steps
