"""CPU-only checks of the packed match-stream layouts (csrc/ggs_layout.cuh) without a GPU:

* `pdb_debug_pack_layout` (the packer's own fill code) places every coordinate where `layout_float_index` says,
  padding rows are zero, segments of the paired layout start at even rounds;
* the GGS kernel's stage-1 traversal -- CTA / warp partition functions shared with the kernel, segment switches, the
  ring / resident / register-stream walks with their fast-path conditions -- replayed sequentially by
  tests/host/geom_host.cu consumes every match exactly once, in the right pair segment, for both layouts, and the per-segment
  sums agree between the layouts.

The parallel execution (shuffles, mbarriers, atomics) is covered by the -m gpu tests only.
"""
import ctypes
import os

import numpy as np
import pytest

from conftest import ROOT
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn


@pytest.fixture(scope="module")
def harness():
    import __graft_entry__ as entry

    entry.build()
    lib = ctypes.CDLL(os.path.join(ROOT, "build", "libgeom_host.so"))
    lib.layout_float_index_host.restype = ctypes.c_longlong
    lib.layout_float_index_host.argtypes = [ctypes.c_longlong, ctypes.c_longlong, ctypes.c_int, ctypes.c_int]
    lib.ggs_host_walk.restype = ctypes.c_int
    lib.ggs_host_walk.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_longlong, ctypes.c_int, ctypes.c_int,
                                  ctypes.c_int, ctypes.c_void_p, ctypes.c_float, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p]
    return lib


def _tiny_segments(frames=6, seed=3):
    """Many short pair segments (1..5 matches) -- more than the kernel's 128-segment chunk when one CTA owns them all."""
    rng = np.random.default_rng(seed)
    pairs = [(a, b) for a in range(frames) for b in range(frames) if a != b] * 6
    counts = rng.integers(1, 6, size=len(pairs))
    i12 = np.concatenate([np.tile(np.array([p], dtype=np.int64), (c, 1)) for p, c in zip(pairs, counts)])
    kp = rng.uniform(0, 224, size=(len(i12), 4))
    return {"kp1": kp[:, :2], "kp2": kp[:, 2:], "i12": i12, "img_shape": (frames, 3, 224, 224)}


CASES = {
    "uniform_64x": lambda: syn.uniform_matches(5, 256, seed=1),          # whole units only: no padding in either layout
    "uniform_odd": lambda: syn.uniform_matches(5, 70, seed=2),            # 70 = 2 rounds + 6 rows: padding in both layouts
    "uniform_33": lambda: syn.uniform_matches(4, 33, seed=3),             # second round of every unit is almost all padding
    "ragged": lambda: syn.scene_matches(7, 150, seed=4, ordered=False, ragged=True)[0],  # hloc-like: 0..300 per unordered pair
    "tiny": _tiny_segments,
    "single_match": lambda: {"kp1": np.array([[1.0, 2.0]]), "kp2": np.array([[3.0, 4.0]]), "i12": np.array([[0, 1]]),
                             "img_shape": (2, 3, 224, 224)},
}


def _segment_rows(m):
    i12 = np.asarray(m["i12"])
    change = np.flatnonzero((i12[1:] != i12[:-1]).any(1)) + 1
    starts = np.concatenate([[0], change])
    return starts, np.diff(np.concatenate([starts, [len(i12)]]))


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("layout", ["plain", "paired"])
def test_packer_places_every_coordinate_where_the_layout_function_says(harness, case, layout):
    m = CASES[case]()
    segs, pts = _native.pack_layout_host(m, layout)
    starts, counts = _segment_rows(m)
    assert np.array_equal(segs[:, 1], counts)
    assert np.array_equal(segs[:, 2:], np.asarray(m["i12"])[starts])  # pair / frame indexing bit-exact
    paired = layout == "paired"
    per_seg = (counts + 63) // 64 * 2 if paired else (counts + 31) // 32
    assert np.array_equal(segs[:, 0], np.concatenate([[0], np.cumsum(per_seg)[:-1]]))
    assert len(pts) == int(per_seg.sum()) * 32
    if paired:
        assert not (segs[:, 0] & 1).any()
    want = np.concatenate([m["kp1"], m["kp2"]], 1).astype(np.float32)  # fp64 -> fp32 rounding of the reference's `.float()` (:167)
    flat = pts.reshape(-1)
    seen = np.zeros(flat.shape, dtype=bool)
    for s, (first_round, count) in enumerate(segs[:, :2]):
        for k in range(count):
            for comp in range(4):
                idx = harness.layout_float_index_host(int(first_round), k, comp, int(paired))
                assert not seen[idx]
                seen[idx] = True
                assert flat[idx] == want[starts[s] + k, comp]
    assert seen.sum() == 4 * len(want)
    assert (flat[~seen] == 0).all()  # padding rows are zero in both layouts


def _walk(harness, m, layout, mode, cpp, seed=0):
    segs, pts = _native.pack_layout_host(m, layout)
    nseg, rounds = len(segs), len(pts) // 32
    segs_s = np.concatenate([segs, np.array([[rounds, 0, 0, 0]], dtype=np.int32)])
    F = np.random.default_rng(seed).normal(scale=1e-3, size=(nseg, 9)).astype(np.float32)
    acc = np.zeros((nseg, 12), np.float32)
    visits = np.zeros(len(m["i12"]), np.int32)
    fast = np.zeros(2, np.int64)
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = harness.ggs_host_walk(P(np.ascontiguousarray(pts)), P(segs_s), nseg, rounds, cpp, int(layout == "paired"), mode, P(F),
                               ctypes.c_float(10.0), P(acc), P(visits), P(fast))
    return rc, acc, visits, fast


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("mode", [0, 1, 2], ids=["resident", "ring", "stream"])
@pytest.mark.parametrize("cpp", [1, 3, 132, 148])
def test_kernel_traversal_consumes_every_match_once_in_both_layouts(harness, case, mode, cpp):
    m = CASES[case]()
    out = {}
    for layout in ("plain", "paired"):
        rc, acc, visits, fast = _walk(harness, m, layout, mode, cpp)
        assert rc == 0, f"{layout}: traversal invariant {rc} violated"
        assert (visits == 1).all(), f"{layout}: matches consumed {np.unique(visits)} times"
        assert fast.sum() == len(visits)
        out[layout] = (acc, fast)
    (a0, f0), (a1, f1) = out["plain"], out["paired"]
    assert np.array_equal(a0[:, 11], a1[:, 11])  # valid counts per pair segment: exact
    scale = np.abs(a0).max(0, keepdims=True) + 1e-30
    np.testing.assert_allclose(a1 / scale, a0 / scale, rtol=0, atol=2e-5)  # same terms, different summation order


def test_paired_layout_keeps_the_packed_fast_path_share_at_benchmark_shape(harness):
    """At the headline shape (config 3: 20 frames, 2048 matches for each of the 380 ordered pairs, 132 CTAs = one per H100 SM) the paired walk
    must take the packed fast path at least as often as the plain one (otherwise the layout would trade MOVs for scalar tails)."""
    m = syn.uniform_matches(20, 2048, seed=5)
    for mode, floor in ((0, 0.99), (1, 0.75)):
        _, _, _, f_plain = _walk(harness, m, "plain", mode, 132)
        _, _, _, f_pair = _walk(harness, m, "paired", mode, 132)
        assert f_pair[0] >= f_plain[0]
        assert f_pair[0] >= floor * f_pair.sum()


def test_layout_probe_rejects_bad_input():
    m = syn.uniform_matches(3, 4, seed=0)
    bad = dict(m)
    bad["i12"] = m["i12"].copy()
    bad["i12"][2, 0] = 3  # frame index outside [0, frames)
    with pytest.raises(ValueError):
        _native.pack_layout_host(bad, "plain")
    with pytest.raises(KeyError):
        _native.pack_layout_host(m, "transposed")
    empty = {"kp1": np.zeros((0, 2)), "kp2": np.zeros((0, 2)), "i12": np.zeros((0, 2), np.int64), "img_shape": (4, 3, 224, 224)}
    for layout in ("plain", "paired"):
        segs, pts = _native.pack_layout_host(empty, layout)
        assert segs.shape == (0, 4) and pts.shape == (0, 4)
