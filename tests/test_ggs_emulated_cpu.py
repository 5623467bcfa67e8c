"""CPU execution of the GGS KERNEL SOURCE (csrc/ggs.cuh, the file nvcc compiles for sm_90a) through the emulation of the CUDA
execution model in tests/host/cuda_emu.h: every CUDA thread is a coroutine, warp collectives / block barriers / the mbarrier
+ bulk-copy ring / the grid-wide release-acquire barrier behave as on the device, CTAs run as concurrent OS threads.

This is test infrastructure for code written without GPU access: it runs both stream layouts (`kPaired` false / true), the
evaluation and the optimisation instantiation (`kEval`), and the three ways stage 1 reads matches (shared-memory resident,
bulk-async ring, register stream) against the reference fixtures (tests/golden, produced by the reference's own modules) and
the fp64 closed form -- same tolerances as the GPU parity tests.  It proves functional correctness of the kernel logic, not
performance and not the absence of device-only hazards (those stay with the -m gpu tests and compute-sanitizer).
"""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT, load_golden, matches_from
from oracle import sampson_f64 as s64
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

MODES = {"resident": (0, 0), "ring": (1, 0), "stream": (1, 1)}  # (force_stream, no_ring)
FLAGS = ((1, 1, 1), (0, 0, 1), (1, 0, 0), (0, 1, 0))


@pytest.fixture(scope="module")
def emu():
    import __graft_entry__ as entry

    entry.build()  # the packer (layout image) lives in the product library, the emulated kernel in build/libkernels_emu.so
    lib = C.CDLL(entry.build_emulator())
    lib.ggs_emu_run.restype = C.c_int
    return lib


def run_kernel(lib, m, pose, layout, mode="resident", cpp=2, eval_flags=None, cfg=None):
    """eval_flags = (R, T, FL): one compute_sampson_distance + backward (kEval); None: the five GGS phases (cfg = GGS_cfg)."""
    segs, pts = _native.pack_layout_host(m, layout)
    rounds = len(pts) // 32
    segs_s = np.concatenate([segs.reshape(-1, 4), np.array([[rounds, 0, 0, 0]], np.int32)])
    N, _, H, W = (int(v) for v in m["img_shape"])
    pose = np.ascontiguousarray(pose, np.float32).reshape(N, 9).copy()
    grad, sc = np.zeros((N, 9), np.float32), np.zeros(4, np.float32)
    nseg = len(segs)
    Fd, Gd = np.zeros((max(nseg, 1), 9), np.float32), np.zeros((max(nseg, 1), 9), np.float32)
    stats = np.zeros(1, _native.GGS_STATS_DTYPE)
    if eval_flags is not None:
        iters, flags = [1], [(1 if eval_flags[0] else 0) | (2 if eval_flags[1] else 0) | (4 if eval_flags[2] else 0)]
        k = dict(alpha=1e-4, lr=1e-2, smax=10.0, momentum=0.9, min_matches=0.0)
    else:
        n = int(cfg["iter_num"])
        iters, flags = [2 * n, n, n, n, 2 * n], [7, 4, 1, 2, 7]  # geometry_guided_sampling.py:47-64, :86-87
        k = dict(alpha=cfg["alpha"], lr=cfg["learning_rate"], smax=cfg["sampson_max"], momentum=0.9, min_matches=cfg["min_matches"])
    it = np.array(iters + [0] * (5 - len(iters)), np.int32)
    fl = np.array(flags + [0] * (5 - len(flags)), np.int32)
    got_mode = C.c_int(-1)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    fs, nr = MODES[mode]
    rc = lib.ggs_emu_run(P(np.ascontiguousarray(pts)), P(segs_s), nseg, rounds, C.c_longlong(len(m["kp1"])), N, C.c_float(H), C.c_float(W),
                         P(pose), int(layout == "paired"), int(eval_flags is not None), cpp, fs, nr, P(it), P(fl), len(iters),
                         C.c_float(k["alpha"]), C.c_float(k["lr"]), C.c_float(k["smax"]), C.c_float(k["momentum"]), C.c_double(k["min_matches"]),
                         P(grad), P(sc), P(Fd), P(Gd), P(stats), C.byref(got_mode))
    assert rc == 0
    assert got_mode.value == {"resident": 0, "ring": 1, "stream": 2}[mode]
    return dict(pose=pose, grad=grad, scalars=sc, F=Fd, G=Gd, stats=stats[0])


def nan_close(actual, desired, atol):
    actual, desired = np.asarray(actual, dtype=np.float64), np.asarray(desired, dtype=np.float64)
    assert np.array_equal(np.isnan(actual), np.isnan(desired))
    ok = ~np.isnan(desired)
    np.testing.assert_allclose(actual[ok], desired[ok], rtol=0, atol=atol)


@pytest.mark.parametrize("layout", ["plain", "paired"])
@pytest.mark.parametrize("mode", sorted(MODES))
@pytest.mark.parametrize("tag", ["scene6", "ragged5", "uniform5", "empty5", "diag4", "clamp4"])
def test_emulated_sampson_eval_vs_reference(emu, tag, mode, layout):
    """compute_sampson_distance + backward through the kernel: valid counts exact, gradient within the GPU test's tolerances,
    including the reference's quirks (NaN poisoning by a diagonal pair, empty valid set, saturated focal clamp)."""
    g = load_golden("sampson.npz")
    m = matches_from(g, tag)
    for flags in FLAGS if mode == "resident" else FLAGS[:1]:
        key = f"{tag}_f{''.join(map(str, flags))}"
        r = run_kernel(emu, m, g[f"{tag}_pose"], layout, mode, cpp=3, eval_flags=flags)
        n_ref = int(g[f"{key}_n_valid"])
        assert int(r["scalars"][1]) == n_ref
        nan_close(r["scalars"][2], g[f"{key}_logged"], 1e-5 * 10)
        if n_ref == 0:
            continue
        ref = g[f"{key}_grad"]
        gmax = np.nanmax(np.abs(ref))
        np.testing.assert_allclose(r["scalars"][0], g[f"{key}_loss"], rtol=2e-5)
        nan_close(r["grad"], ref, 2e-4 * gmax)
        c = s64.sampson_closed_form_f64(g[f"{tag}_pose"], m, *map(bool, flags))
        nan_close(r["grad"], c["grad"], 1e-4 * gmax)
        assert np.array_equal(r["grad"] == 0, ref == 0)


@pytest.mark.parametrize("layout", ["plain", "paired"])
@pytest.mark.parametrize("mode,cpp", [("resident", 2), ("ring", 3), ("stream", 1)])
@pytest.mark.parametrize("tag", ["scene5", "scene8"])
def test_emulated_five_phase_ggs_vs_reference(emu, tag, mode, cpp, layout):
    """geometry_guided_sampling (5 x GGS_optimize: clip, momentum, phase flags) through the optimisation instantiation of the
    kernel, several CTAs synchronising through the grid barrier: pose within 2e-5 of the reference's own output."""
    g = load_golden("ggs.npz")
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = int(g["iter_num"])
    r = run_kernel(emu, matches_from(g, tag), g[f"{tag}_pose"], layout, mode, cpp=cpp, cfg=cfg)
    ref = g[f"{tag}_out"]
    # GPU tolerance 2e-5.  scene8 holds one match whose Sampson error sits on the validity threshold: whether it counts depends on
    # the summation order of the cross-CTA atomics (OS-thread interleaving here) and moves the pose by 1.4e-5 -> twice that bound
    np.testing.assert_allclose(r["pose"], ref, rtol=0, atol=4e-5 * np.abs(ref).max())
    n = cfg["iter_num"]
    assert list(r["stats"]["iters"]) == [2 * n, n, n, n, 2 * n]
    assert int(r["stats"]["dropped"].sum()) == int(g[f"{tag}_drops"])
    np.testing.assert_allclose(r["stats"]["sampson"], g[f"{tag}_log"], rtol=2e-3)


@pytest.mark.parametrize("layout", ["plain", "paired"])
def test_emulated_early_exit_vs_reference(emu, layout):
    """`len(valid) / N < min_matches` ends every phase before its first update (:103-108): the pose comes back bit-identical."""
    g = load_golden("ggs.npz")
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = int(g["iter_num"])
    r = run_kernel(emu, matches_from(g, "drop"), g["drop_pose"], layout, "resident", cpp=2, cfg=cfg)
    assert int(r["stats"]["dropped"].sum()) == int(g["drop_drops"]) == 5
    assert np.array_equal(r["pose"], g["drop_out"].reshape(r["pose"].shape))


@pytest.mark.parametrize("mode,cpp", [("resident", 4), ("ring", 2), ("stream", 1)])
def test_emulated_layouts_agree_on_ragged_and_tiny_segments(emu, mode, cpp):
    """hloc-like ragged pair sizes and single-match segments (more than 128 segments per CTA with cpp = 1 -> multi-chunk
    walk): the paired layout gives the same statistics as the plain one and the fp64 closed form."""
    from test_layout_cpu import _tiny_segments

    for m, pose in ((syn.scene_matches(7, 150, seed=4, ordered=False, ragged=True)[0], syn.scene_matches(7, 2, seed=4)[2]),
                    (_tiny_segments(), syn.scene_matches(6, 2, seed=3)[2])):
        out = {lay: run_kernel(emu, m, pose, lay, mode, cpp=cpp, eval_flags=(1, 1, 1)) for lay in ("plain", "paired")}
        assert out["plain"]["scalars"][1] == out["paired"]["scalars"][1]
        c = s64.sampson_closed_form_f64(pose, m)
        assert abs(int(out["paired"]["scalars"][1]) - c["n_valid"]) <= 2
        if c["n_valid"] == 0:
            continue
        gmax = np.abs(c["grad"]).max()
        for lay in out:
            np.testing.assert_allclose(out[lay]["grad"], c["grad"], rtol=0, atol=3e-4 * gmax)
        assert np.array_equal(out["plain"]["F"], out["paired"]["F"])  # F' of every segment does not depend on the layout


@pytest.mark.parametrize("layout", ["plain", "paired"])
@pytest.mark.parametrize("cpp,group,xch", [(5, 2, 0), (7, 3, 0), (6, 6, 0), (7, 3, 1)])
def test_emulated_exchange_modes(emu, layout, cpp, group, xch, monkeypatch):
    """The per-iteration all-reduce of the partial gradients.  xch = 0: flag-carrying exchange words (csrc/common.cuh st_ll /
    ll_sum) -- groups of `group` CTAs with a ragged last group (two levels), or every CTA reading every slot (group == cpp);
    xch = 1 (the default everywhere else in this file): one hop through {sum, arrivals} vector reductions.  Same fixtures and
    tolerances as the runs above."""
    monkeypatch.setenv("PDB_GGS_GROUP", str(group))
    monkeypatch.setenv("PDB_GGS_XCH", str(xch))
    g = load_golden("ggs.npz")
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = int(g["iter_num"])
    m = matches_from(g, "scene5")
    r = run_kernel(emu, m, g["scene5_pose"], layout, "resident", cpp=cpp, cfg=cfg)
    ref = g["scene5_out"]
    np.testing.assert_allclose(r["pose"], ref, rtol=0, atol=2e-5 * np.abs(ref).max())
    n = cfg["iter_num"]
    assert list(r["stats"]["iters"]) == [2 * n, n, n, n, 2 * n]
    # evaluation instantiation through the same exchange
    key = "scene6_f111"
    gs = load_golden("sampson.npz")
    e = run_kernel(emu, matches_from(gs, "scene6"), gs["scene6_pose"], layout, "resident", cpp=cpp, eval_flags=(1, 1, 1))
    assert int(e["scalars"][1]) == int(gs[f"{key}_n_valid"])
    nan_close(e["grad"], gs[f"{key}_grad"], 2e-4 * np.nanmax(np.abs(gs[f"{key}_grad"])))
