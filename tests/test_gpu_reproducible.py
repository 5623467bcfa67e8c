"""Reproducible sampling on the GPU: with `torch.use_deterministic_algorithms(True)` every sampling entry returns the same bits on
every call (pdb_set_reproducible, DESIGN.md section 4.1 / 4.3), and its results stay within the tolerances the default kernels
are held to.

Tolerances, stated once:
  * five-phase GGS pose (iter_num = 5): 3e-5 * max|pose| against `po.geometry_guided_sampling`, as
    tests/test_gpu_fullsize.py at config-3 size;
  * tensor-core engine steps: 5e-3 * max(1, max|out|) against the float64 step from the device's own state, as
    tests/test_gpu_ddim.py for that engine.

torch's switch is process-global: every test restores it.
"""
import re
from contextlib import contextmanager
from functools import partial

import numpy as np
import pytest
import torch

import ddim_oracle as dd
from conftest import load_golden
from oracle import pose_oracle as po
from oracle.denoiser_f64 import DenoiserF64

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


@contextmanager
def deterministic(on: bool = True):
    before, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(on)
    try:
        yield
    finally:
        torch.use_deterministic_algorithms(before, warn_only=warn)
        # the context is shared with every other test module, some of which call entries that do not mirror the switch
        _native.Context.get(torch.device("cuda:0"))._sync_reproducible()


def pack(ctx, m, layout):
    before = ctx.ggs_layout
    ctx.set_ggs_layout(layout)
    try:
        return ctx.pack_matches(m)
    finally:
        ctx.set_ggs_layout(before)  # the context is shared with every other test module


def bits(t):
    return t.detach().cpu().numpy().tobytes() if torch.is_tensor(t) else np.asarray(t).tobytes()


def ggs_cfg(iter_num=5):
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=iter_num, verbose=False)
    return cfg


def ggs_kernels(fn):
    """Names of the GGS kernels `fn` launches."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.name for e in prof.events() if "ggs_entry" in e.name]


@pytest.fixture(scope="module")
def cfg3():
    """Config 3: 20 frames x 380 ordered pairs x 2048 matches (778 240), resident slices, 132 CTAs: two-level slot exchange."""
    m, _, start = syn.scene_matches(20, 2048, seed=77)
    return m, start, po.geometry_guided_sampling(torch.from_numpy(start)[None], 5, m, ggs_cfg())[0].numpy()


@pytest.fixture(scope="module")
def small():
    m, _, start = syn.scene_matches(12, 256, seed=12)
    return m, start, po.geometry_guided_sampling(torch.from_numpy(start)[None], 5, m, ggs_cfg())[0].numpy()


@pytest.mark.parametrize("layout", ["plain", "paired"])
@pytest.mark.parametrize("case", ["cfg3_resident", "cfg3_streamed", "ragged_groups"])
def test_ggs_same_bits_every_call(ctx, dev, cfg3, small, case, layout, monkeypatch):
    """geometry_guided_sampling three times: the same pose and statistics bits, within the oracle tolerance."""
    if case == "cfg3_streamed":
        monkeypatch.setenv("PDB_GGS_FORCE_STREAM", "1")  # the bulk-async ring instead of the resident slice
    if case == "ragged_groups":  # 17 CTAs in exchange groups of 5 (5 + 5 + 5 + 2): more CTAs than a group, ragged last group
        monkeypatch.setenv("PDB_GGS_CPP", "17")
        monkeypatch.setenv("PDB_GGS_GROUP", "5")
    m, start, want = small if case == "ragged_groups" else cfg3
    pm = pack(ctx, m, layout)
    runs = []
    with deterministic():
        for _ in range(3):
            pose = torch.from_numpy(start)[None].to(dev).clone()
            stats = ctx.ggs([pm], pose, ggs_cfg())
            runs.append((bits(pose), bits(stats), pose[0].cpu().numpy(), _native.stats_to_numpy(stats)[0]))
    assert all(r[0] == runs[0][0] and r[1] == runs[0][1] for r in runs[1:])
    got, st = runs[0][2], runs[0][3]
    np.testing.assert_allclose(got, want, rtol=0, atol=3e-5 * np.abs(want).max())
    assert list(st["iters"]) == [10, 5, 5, 5, 10] and int(st["dropped"].sum()) == 0


def test_dispatch_follows_the_switch(ctx, dev, cfg3):
    """Switch on: the reproducible kernel; off again: the default dispatch (the lean kernel at config 3).  A refused setter value
    changes nothing and leaves the context usable."""
    m, start, _ = cfg3
    pm = pack(ctx, m, "paired")

    def call():
        pose = torch.from_numpy(start)[None].to(dev).clone()
        ctx.ggs([pm], pose, ggs_cfg(1))
        return pose

    lean = re.compile(r"ggs_entry<false, (true|false), false, true>")
    with deterministic(False):
        call()  # mirror the switch (off) into the library before profiling
        assert any(lean.search(n) for n in ggs_kernels(call))
    with deterministic():
        first = call()
        names = ggs_kernels(call)
        assert names and all("ggs_entry_repro" in n for n in names)
        assert ctx.lib.pdb_set_reproducible(ctx.handle, 2) == _native.PDB_ERR_INVALID
        assert ctx.lib.pdb_set_reproducible(ctx.handle, -1) == _native.PDB_ERR_INVALID
        again = call()  # still reproducible, still working
        assert bits(again) == bits(first)
    with deterministic(False):
        names = ggs_kernels(call)
        assert names and all(lean.search(n) for n in names)


def _guided_setup(dev, frames=20, per_pair=2048):
    state = syn.random_denoiser_state(5, 0.05)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    dif = pdb.GaussianDiffusion()
    dif.model = den
    dif = dif.to(dev)
    m, _, _ = syn.scene_matches(frames, per_pair, seed=31)
    cond = partial(pdb.geometry_guided_sampling, matches_dict=m, GGS_cfg=ggs_cfg(100))
    return dif, cond, syn.random_features(1, frames, 31).to(dev)


def test_sample_with_ggs_same_bits(dev):
    """sample() with GGS on (10 guided steps of 700 inner iterations) at 20 frames, twice from the same seed."""
    dif, cond, z = _guided_setup(dev)
    runs = []
    with deterministic():
        for _ in range(2):
            torch.manual_seed(0)
            pose, trail = dif.sample([1, 20, 9], z, cond_fn=cond, cond_start_step=10)
            runs.append((bits(trail), bits(dif.last_ggs_stats)))
    assert runs[0] == runs[1]
    assert torch.isfinite(trail).all()


def test_ddim_guided_steps_same_bits(dev):
    """ddim_sample with guided_steps = 2 (two DDIM jumps over the guided tail, GGS after each), twice with the same draws."""
    dif, cond, z = _guided_setup(dev)
    draws = torch.randn(1, 1, 20, 9, generator=torch.Generator().manual_seed(4)).to(dev)
    runs = []
    with deterministic():
        for _ in range(2):
            pose, trail = dif.ddim_sample([1, 20, 9], z, cond_fn=cond, cond_start_step=10, sampling_timesteps=12, eta=0.0,
                                          draws=draws, guided_steps=2)
            runs.append((bits(trail), bits(dif.last_ggs_stats)))
    assert runs[0] == runs[1]
    assert trail.shape == (13, 1, 20, 9) and torch.isfinite(trail).all()


@pytest.mark.parametrize("B,N", [(8, 20), (1, 128)], ids=["8x20", "1x128"])
def test_tc_engine_same_bits_and_within_f64_bound(dev, B, N):
    """The tensor-core engine unguided (DDIM, 20 steps, eta = 1): two runs with the same draws give the same trail, and every step
    is within the engine's float64 bound."""
    g = load_golden("denoiser.npz")
    state = syn.random_denoiser_state(int(g["weight_seed"]), float(g["bias_std"]))
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    den = den.to(dev)
    ctx = den.native_context()
    k, eta = 20, 1.0
    z = syn.random_features(B, N, 3)
    draws = torch.randn(1 + k, B, N, 9, generator=torch.Generator().manual_seed(5))
    ctx.set_denoiser_engine("tf32")
    try:
        with deterministic():
            trails = [ctx.sample_loop_ddim(z.to(dev), draws.to(dev), k, eta, None, None, 0)[1] for _ in range(2)]
    finally:
        ctx.set_denoiser_engine("auto")  # the context is shared with every other test module
    assert bits(trails[0]) == bits(trails[1])
    ref = DenoiserF64(state)
    trail = trails[0].cpu()
    for i, (t, s, _c) in enumerate(dd.prefix_steps(k, 0, eta)):
        want, _, _, _ = dd.ddim_step_f64(ref, trail[i], t, s, eta, z, draws[1 + i])
        lim = 5e-3 * max(1.0, want.abs().max().item())
        assert (trail[1 + i].double() - want).abs().max().item() <= lim, (i, t)
