"""CPU execution of the fp32 denoiser kernel source (csrc/denoiser.cuh) at every token-tile width it is compiled for, through the
execution-model emulation of tests/host/cuda_emu.h (see tests/test_denoiser_emulated_cpu.py), at the evaluation's sequence length
of 10 frames.

Every output of a linear stage has exactly one owner, and its k-slice order, warp exchange and cross-warp sum do not depend on the
tile width TS; attention and the tail are per sequence / per token.  So eps is bit-identical across TS in {8, 16, 20, 24, 32} and
across both stage hand-overs, and a sequence's eps does not depend on the batch it is part of.  Each run is also held to the float64
bound of the device tests: max |eps - eps_f64| <= 4 * d32 + 1e-6, d32 = the fp32 oracle's own distance to float64
(oracle/denoiser_f64.py).  Kernel logic only: register allocation, unrolling and launch geometry of the device build are checked by
tests/test_gpu_denoiser_tiles.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle.denoiser_f64 import DenoiserF64, bound
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn
from test_denoiser_emulated_cpu import run_steps

TILES = (8, 16, 20, 24, 32)
T_STEP = 37


@pytest.fixture(scope="module")
def emu():
    import __graft_entry__ as entry

    entry.build()
    lib = C.CDLL(entry.build_emulator())
    lib.denoiser_emu_run.restype = C.c_int
    return lib


@pytest.fixture(scope="module")
def golden_state():
    g = load_golden("denoiser.npz")
    return syn.random_denoiser_state(int(g["weight_seed"]), float(g["bias_std"]))


@pytest.fixture(scope="module")
def weights(golden_state):
    tensors = [np.ascontiguousarray(golden_state[name].numpy(), dtype=np.float32) for name in syn.denoiser_param_shapes()]
    assert len(tensors) == _native.PDB_NUM_WEIGHT_TENSORS
    return tensors


@pytest.fixture(scope="module")
def case(golden_state):
    """Two 10-frame sequences; the first is also run alone.  eps in float64 and d32 for both shapes."""
    gen = torch.Generator().manual_seed(10)
    x = torch.randn(2, 10, 9, generator=gen)
    z = torch.randn(2, 10, 384, generator=gen)
    ref = DenoiserF64(golden_state)
    alone = ref.noise_f64(x[:1], T_STEP, z[:1])
    pair = ref.noise_f64(x, T_STEP, z)
    return dict(x=x.numpy(), z=z.numpy(), f64={1: alone, 2: pair})


_runs = {}


def emulated(emu, weights, case, monkeypatch, batch, handover, ts, grid):
    key = (batch, handover, ts, grid)
    if key not in _runs:
        monkeypatch.setenv("PDB_DEN_FLAG", "1" if handover == "flags" else "0")  # read by tests/host/kernels_emu.cpp per run
        r = run_steps(emu, weights, case["x"][:batch], case["z"][:batch], T_STEP, T_STEP, grid=grid, token_tile=ts)
        _runs[key] = r["eps"]
    return _runs[key]


def check_f64(eps, case, batch):
    eps64, d32 = case["f64"][batch]
    err = np.abs(eps.astype(np.float64) - eps64.numpy()).max()
    assert err <= bound(d32) and bound(d32) <= 3e-5, (err, d32)
    return err


@pytest.mark.parametrize("ts", TILES)
@pytest.mark.parametrize("handover", ["barriers", "flags"])
def test_emulated_10_frames_every_token_tile(emu, weights, case, monkeypatch, handover, ts):
    """1 x 10 frames: TS 16 is what pick_token_tile chooses; 8, 20, 24 and 32 leave 6, 10, 14 and 22 padded rows.  Grids of 3 to 7
    CTAs.  eps within the float64 bound, and bit-identical to the barrier-mode TS 16 run."""
    eps = emulated(emu, weights, case, monkeypatch, 1, handover, ts, 3 + TILES.index(ts))
    check_f64(eps, case, 1)
    want = emulated(emu, weights, case, monkeypatch, 1, "barriers", 16, 4)
    assert np.array_equal(eps, want)


@pytest.mark.parametrize("ts", [16, 24])
def test_emulated_two_sequences_cut_by_tile_boundary(emu, weights, case, monkeypatch, ts):
    """2 x 10 frames, barrier mode: with TS 16 the second sequence straddles the tile boundary at token 16 (and the second tile
    has 12 padded rows); with TS 24 both share one tile with 4 padded rows.  Within the float64 bound, equal across the two widths,
    and the first sequence equals its own 1 x 10 run bit for bit."""
    eps = emulated(emu, weights, case, monkeypatch, 2, "barriers", ts, 5)
    check_f64(eps, case, 2)
    assert np.array_equal(eps[:1], emulated(emu, weights, case, monkeypatch, 1, "barriers", 16, 4))
    if ts == 24:
        assert np.array_equal(eps, emulated(emu, weights, case, monkeypatch, 2, "barriers", 16, 5))
