"""CPU execution of the fp32 denoiser kernel source on DDIM steps (csrc/denoiser.cuh through tests/host/cuda_emu.h, both stage
hand-overs).  pdb_sample_loop_ddim runs the DDIM prefix as the kernel's DDPM loop over per-timestep tables whose rows are the
DDIM step's: here a 3-step, eta = 0.5 prefix, one emulated launch per step with the step's coefficient row in the schedule slot
of its timestep and its draw in that timestep's draw slot, each step fed the kernel's own previous output and checked against the
fp32 oracle's DDIM step (tests/ddim_oracle.py) with the tolerance of the emulated p_sample test."""
import ctypes as C

import numpy as np
import pytest
import torch

import ddim_oracle as dd
from conftest import load_golden
from oracle import pose_oracle as po
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn


@pytest.fixture(scope="module")
def emu():
    import __graft_entry__ as entry

    entry.build()
    lib = C.CDLL(entry.build_emulator())
    lib.denoiser_emu_run.restype = C.c_int
    return lib


@pytest.fixture(autouse=True, params=["flags", "barriers"])
def handover(request, monkeypatch):
    monkeypatch.setenv("PDB_DEN_FLAG", "1" if request.param == "flags" else "0")  # read by tests/host/kernels_emu.cpp per run
    return request.param


@pytest.fixture(scope="module")
def weights():
    g = load_golden("denoiser.npz")
    state = syn.random_denoiser_state(int(g["weight_seed"]), float(g["bias_std"]))
    tensors = [np.ascontiguousarray(state[name].numpy(), dtype=np.float32) for name in syn.denoiser_param_shapes()]
    return state, tensors


@pytest.mark.parametrize("g", [0, 10])
def test_emulated_ddim_prefix_vs_oracle(emu, weights, g):
    state, tensors = weights
    k, eta, B, N = 3, 0.5, 1, 20
    S = B * N
    steps_t, coef = _native.ddim_table(k + g, g, eta)
    sched = _native.schedule_table()
    gp = load_golden("p_sample.npz")
    z = np.ascontiguousarray(gp["z"], np.float32).reshape(S, 384)
    rng = np.random.default_rng(3 + g)
    draws = rng.normal(size=(1 + k, S, 9)).astype(np.float32)
    arr = (C.c_void_p * len(tensors))(*[t.ctypes.data for t in tensors])
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    net = po.build_denoiser(state)
    zt = torch.from_numpy(z).reshape(B, N, 384)
    x = draws[0].copy()
    for i, (t, s, c) in enumerate(dd.prefix_steps(k, g, eta)):
        assert steps_t[i] == t and coef[i, 5] == s
        table = sched.copy()
        table[t] = coef[i]  # the DDIM row where the kernel reads timestep t's row
        slots = np.zeros((101, S, 9), np.float32)
        slots[1 + (99 - t)] = draws[1 + i]
        trail = np.zeros((101, S, 9), np.float32)
        eps, x0, mean = (np.zeros((S, 9), np.float32) for _ in range(3))
        xin = x.copy()
        rc = emu.denoiser_emu_run(arr, P(table), B, N, t, t, g, P(x), P(z), P(slots), P(trail), P(eps), P(x0), P(mean), 3, 20)
        assert rc == 0
        want, want_x0 = dd.ddim_step(net, torch.from_numpy(xin).reshape(B, N, 9), t, zt, c, torch.from_numpy(draws[1 + i]).reshape(B, N, 9))
        want, want_x0 = want.reshape(S, 9).numpy(), want_x0.reshape(S, 9).numpy()
        np.testing.assert_allclose(x, want, rtol=0, atol=2e-5 * np.abs(want).max() + 1e-5)
        b_t = float(coef[i, 1])
        np.testing.assert_allclose(x0, want_x0, rtol=0, atol=1e-5 * np.abs(want_x0).max() + 3e-5 * b_t)
