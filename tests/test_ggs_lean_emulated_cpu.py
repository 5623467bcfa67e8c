"""CPU execution of the lean GGS instantiation (`ggs_body<false, kPaired, false, true>`, csrc/ggs.cuh) through the emulation of
the CUDA execution model (tests/host/cuda_emu.h), and of the rule that selects it: shared-memory-resident slices, at most
kGgsMaxSeg = 128 pair segments per CTA (`ggs_lean_fits`), the one-hop exchange, optimisation only.

Same fixtures and tolerances as tests/test_ggs_emulated_cpu.py.  `ggs_emu_run_dispatch` applies the launch rule of
api_core.cu::launch_ggs_chunk and reports which instantiation ran; `ggs_emu_run` always runs the general one.
"""
import ctypes as C

import numpy as np
import pytest

from conftest import load_golden, matches_from
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn
from test_ggs_emulated_cpu import MODES, emu  # noqa: F401  (module fixture: builds the library and the emulator)
from test_layout_cpu import _tiny_segments


def run(lib, m, pose, layout, cpp, cfg=None, eval_flags=None, mode="resident", dispatch=True):
    """One emulated launch; returns (pose, stats, lean) where lean says whether the lean instantiation ran."""
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
        k = dict(alpha=1e-4, lr=1e-2, sampson_max=10.0, min_matches=0.0)
    else:
        n = int(cfg["iter_num"])
        iters, flags = [2 * n, n, n, n, 2 * n], [7, 4, 1, 2, 7]
        k = dict(alpha=cfg["alpha"], lr=cfg["learning_rate"], sampson_max=cfg["sampson_max"], min_matches=cfg["min_matches"])
    it = np.array(iters + [0] * (5 - len(iters)), np.int32)
    fl = np.array(flags + [0] * (5 - len(flags)), np.int32)
    got_mode, lean = C.c_int(-1), C.c_int(-1)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    fs, nr = MODES[mode]
    args = [P(np.ascontiguousarray(pts)), P(segs_s), nseg, rounds, C.c_longlong(len(m["kp1"])), N, C.c_float(H), C.c_float(W), P(pose),
            int(layout == "paired"), int(eval_flags is not None), cpp, fs, nr, P(it), P(fl), len(iters), C.c_float(k["alpha"]),
            C.c_float(k["lr"]), C.c_float(k["sampson_max"]), C.c_float(0.9), C.c_double(k["min_matches"]), P(grad), P(sc), P(Fd), P(Gd),
            P(stats), C.byref(got_mode)]
    if dispatch:
        assert lib.ggs_emu_run_dispatch(*args, C.byref(lean)) == 0
    else:
        assert lib.ggs_emu_run(*args) == 0
        lean.value = 0
    assert got_mode.value == {"resident": 0, "ring": 1, "stream": 2}[mode]
    return pose, stats[0], bool(lean.value)


def golden_cfg(g):
    cfg = syn.default_ggs_cfg()
    cfg["iter_num"] = int(g["iter_num"])
    return cfg


@pytest.mark.parametrize("layout", ["plain", "paired"])
@pytest.mark.parametrize("cpp", [2, 3, 4])
@pytest.mark.parametrize("tag", ["scene5", "scene8"])
def test_lean_five_phase_ggs_vs_reference(emu, tag, cpp, layout):
    """geometry_guided_sampling through the lean instantiation: pose within the tolerance of the general kernel's emulated run
    (twice the GPU's 2e-5, see test_ggs_emulated_cpu.py), the reference's per-phase log and drop count."""
    g = load_golden("ggs.npz")
    cfg = golden_cfg(g)
    pose, stats, lean = run(emu, matches_from(g, tag), g[f"{tag}_pose"], layout, cpp, cfg=cfg)
    assert lean
    ref = g[f"{tag}_out"]
    np.testing.assert_allclose(pose, ref, rtol=0, atol=4e-5 * np.abs(ref).max())
    n = cfg["iter_num"]
    assert list(stats["iters"]) == [2 * n, n, n, n, 2 * n]
    assert int(stats["dropped"].sum()) == int(g[f"{tag}_drops"])
    np.testing.assert_allclose(stats["sampson"], g[f"{tag}_log"], rtol=2e-3)


@pytest.mark.parametrize("layout", ["plain", "paired"])
def test_lean_early_exit_bit_identical(emu, layout):
    """Every phase ends before its first update (:103-108): the lean kernel returns the pose bit-identical."""
    g = load_golden("ggs.npz")
    pose, stats, lean = run(emu, matches_from(g, "drop"), g["drop_pose"], layout, 2, cfg=golden_cfg(g))
    assert lean
    assert int(stats["dropped"].sum()) == int(g["drop_drops"]) == 5
    assert np.array_equal(pose, g["drop_out"].reshape(pose.shape))


@pytest.mark.parametrize("layout", ["plain", "paired"])
@pytest.mark.parametrize("case,cpp", [("ragged", 4), ("tiny", 2), ("tiny", 3)])
def test_lean_agrees_with_general_on_ragged_and_tiny_segments(emu, case, cpp, layout):
    """hloc-like ragged pair sizes and 1..5-match segments: the lean and the general instantiation give the same statistics
    and poses within the emulated tolerance."""
    if case == "ragged":
        m, pose0 = syn.scene_matches(7, 150, seed=4, ordered=False, ragged=True)[0], syn.scene_matches(7, 2, seed=4)[2]
    else:
        m, pose0 = _tiny_segments(), syn.scene_matches(6, 2, seed=3)[2]
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=3, min_matches=0)
    got, st_l, lean = run(emu, m, pose0, layout, cpp, cfg=cfg)
    want, st_g, _ = run(emu, m, pose0, layout, cpp, cfg=cfg, dispatch=False)
    assert lean
    assert list(st_l["iters"]) == list(st_g["iters"]) == [6, 3, 3, 3, 6]
    assert list(st_l["n_valid"]) == list(st_g["n_valid"])
    np.testing.assert_allclose(st_l["sampson"], st_g["sampson"], rtol=1e-5)
    np.testing.assert_allclose(got, want, rtol=0, atol=4e-5 * np.abs(want).max())


def test_lean_dispatch_rule(emu, monkeypatch):
    """The lean instantiation runs exactly when every CTA's slice is resident and holds at most 128 segments, the exchange is
    the one-hop mode and the call optimises; everything else takes the general kernel."""
    g = load_golden("ggs.npz")
    cfg = golden_cfg(g)
    cfg["iter_num"] = 1
    m5, p5 = matches_from(g, "scene5"), g["scene5_pose"]
    tiny, ptiny = _tiny_segments(), syn.scene_matches(6, 2, seed=3)[2]
    assert run(emu, m5, p5, "paired", 2, cfg=cfg)[2]
    assert not run(emu, m5, p5, "paired", 2, eval_flags=(1, 1, 1))[2]          # evaluation
    assert not run(emu, m5, p5, "paired", 2, cfg=cfg, mode="ring")[2]          # slice streamed through the ring
    assert not run(emu, m5, p5, "paired", 1, cfg=cfg, mode="stream")[2]        # register stream
    for lay in ("plain", "paired"):
        assert not run(emu, tiny, ptiny, lay, 1, cfg=cfg)[2]                    # 180 segments in one CTA: two chunks
        assert run(emu, tiny, ptiny, lay, 2, cfg=cfg)[2]                        # at most 128 per CTA
    monkeypatch.setenv("PDB_GGS_XCH", "0")
    assert not run(emu, m5, p5, "paired", 2, cfg=cfg)[2]                       # exchange through flag-carrying slots
