"""CPU execution of the reproducible GGS instantiation (`ggs_body<false, kPaired, false, false, true>`, csrc/ggs.cuh) through the
emulation of the CUDA execution model (tests/host/cuda_emu.h), under different schedules.

`ggs_emu_run_scheduled` (tests/host/ggs_repro_emu.cpp) permutes the order in which the emulator resumes the kernel's warps:
schedule 0 is the emulator's own order, 1 reverses the warps, k >= 2 rotates them by k.  Every floating-point sum of the
reproducible instantiation has a fixed order, so its pose and statistics must come back with the same bits under every
schedule.  The default instantiation, run with the slot exchange so that the cross-CTA sums are fixed too, must change under the
same knob: that shows the knob reaches the order-sensitive shared-memory sums which the reproducible instantiation replaces.

The scene: 34 frames (more than one warp of frames in stage 2b), each frame paired with its three successors (96 segments of one
or two rounds), two CTAs: every warp walks about three segments, and every frame collects adjoints from up to six segments.
"""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import pose_oracle as po
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn
from test_ggs_emulated_cpu import MODES, emu  # noqa: F401  (module fixture: builds the library and the emulator)

ITER_NUM = 1  # 2 + 1 + 1 + 1 + 2 inner iterations


@pytest.fixture(scope="module")
def scene():
    m, _, start = syn.scene_matches(34, 24, seed=91, ordered=False)
    keep = (m["i12"][:, 1] - m["i12"][:, 0]) <= 3
    m = dict(m, kp1=m["kp1"][keep], kp2=m["kp2"][keep], i12=m["i12"][keep])
    cfg = syn.default_ggs_cfg()
    cfg.update(iter_num=ITER_NUM, verbose=False)
    log = []
    want = po.geometry_guided_sampling(torch.from_numpy(start)[None], 5, m, cfg, log=log)[0].numpy()
    return m, start, cfg, want, log


def run(lib, m, pose, cfg, layout, mode, repro, schedule, cpp=2):
    """One emulated five-phase launch of the reproducible (repro = 1) or the default instantiation under `schedule`."""
    segs, pts = _native.pack_layout_host(m, layout)
    rounds = len(pts) // 32
    segs_s = np.concatenate([segs.reshape(-1, 4), np.array([[rounds, 0, 0, 0]], np.int32)])
    N, _, H, W = (int(v) for v in m["img_shape"])
    pose = np.ascontiguousarray(pose, np.float32).reshape(N, 9).copy()
    stats = np.zeros(1, _native.GGS_STATS_DTYPE)
    n = int(cfg["iter_num"])
    it = np.array([2 * n, n, n, n, 2 * n], np.int32)
    fl = np.array([7, 4, 1, 2, 7], np.int32)
    got_mode = C.c_int(-1)
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    fs, nr = MODES[mode]
    rc = lib.ggs_emu_run_scheduled(P(np.ascontiguousarray(pts)), P(segs_s), len(segs), rounds, C.c_longlong(len(m["kp1"])), N,
                                   C.c_float(H), C.c_float(W), P(pose), int(layout == "paired"), cpp, fs, nr, P(it), P(fl), 5,
                                   C.c_float(cfg["alpha"]), C.c_float(cfg["learning_rate"]), C.c_float(cfg["sampson_max"]),
                                   C.c_float(0.9), C.c_double(cfg["min_matches"]), P(stats), C.byref(got_mode), int(repro), schedule)
    assert rc == 0
    assert got_mode.value == {"resident": 0, "ring": 1, "stream": 2}[mode]
    return pose, stats[0]


def same_bits(a, b):
    return np.asarray(a).tobytes() == np.asarray(b).tobytes()


@pytest.mark.parametrize("layout,mode", [("plain", "resident"), ("paired", "ring")])
def test_reproducible_ggs_same_bits_under_every_schedule(emu, scene, layout, mode, monkeypatch):
    monkeypatch.delenv("PDB_GGS_XCH", raising=False)
    m, start, cfg, want, log = scene
    runs = [run(emu, m, start, cfg, layout, mode, repro=True, schedule=s) for s in (0, 1, 5)]
    for pose, stats in runs[1:]:
        assert same_bits(pose, runs[0][0])
        assert same_bits(stats, runs[0][1])
    pose, stats = runs[0]
    # tolerances of test_ggs_emulated_cpu.py's five-phase runs
    np.testing.assert_allclose(pose, want, rtol=0, atol=4e-5 * np.abs(want).max())
    assert list(stats["iters"]) == [e["iters"] for e in log] == [2 * ITER_NUM, ITER_NUM, ITER_NUM, ITER_NUM, 2 * ITER_NUM]
    assert int(stats["dropped"].sum()) == 0
    np.testing.assert_allclose(stats["sampson"], [e["sampson"] for e in log], rtol=2e-3)


def test_default_ggs_changes_under_the_schedule_knob(emu, scene, monkeypatch):
    """The default instantiation's shared-memory atomics add in scheduling order: the same launch gives other bits under another
    schedule (the slot exchange keeps the cross-CTA sums fixed, so the difference comes from inside the CTA)."""
    monkeypatch.setenv("PDB_GGS_XCH", "0")
    m, start, cfg, want, _ = scene
    a, _ = run(emu, m, start, cfg, "plain", "resident", repro=False, schedule=0)
    b, _ = run(emu, m, start, cfg, "plain", "resident", repro=False, schedule=1)
    assert not same_bits(a, b)
    for pose in (a, b):
        np.testing.assert_allclose(pose, want, rtol=0, atol=4e-5 * np.abs(want).max())
