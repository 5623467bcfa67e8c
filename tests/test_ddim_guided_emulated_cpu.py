"""CPU execution of the fp32 denoiser kernel source on a guided DDIM jump (csrc/denoiser.cuh through tests/host/cuda_emu.h, both
stage hand-overs).  pdb_sample_loop_ddim_guided puts guided jump i's coefficient row in the schedule slot of a virtual timestep
v = g'-1-i below guide_below, so the kernel's DDPM update leaves the DDIM mean: no noise although the draws hold some, and no trail
slot written.  The emulator tabulates the time embedding per slot from the loaded weights (the library gathers the real timestep's
block into slot v; that gather is checked on the GPU), so the oracle's network here is evaluated at v."""
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


@pytest.mark.parametrize("g,gs,i", [(10, 5, 0), (10, 3, 2)])
def test_emulated_guided_jump_leaves_the_mean(emu, g, gs, i):
    g_ = load_golden("denoiser.npz")
    state = syn.random_denoiser_state(int(g_["weight_seed"]), float(g_["bias_std"]))
    tensors = [np.ascontiguousarray(state[name].numpy(), dtype=np.float32) for name in syn.denoiser_param_shapes()]
    k, eta, B, N = 4, 0.5, 1, 20
    S = B * N
    _, coef = _native.ddim_table(k + gs, g, eta, guided_steps=gs)
    row = coef[k + i]
    assert row[4] > 0 or row[5] == -1  # a noise scale the kernel must not apply (zero only on the jump to x0)
    v = gs - 1 - i
    table = _native.schedule_table()
    table[v] = row
    gp = load_golden("p_sample.npz")
    z = np.ascontiguousarray(gp["z"], np.float32).reshape(S, 384)
    rng = np.random.default_rng(11 + i)
    x = rng.normal(size=(S, 9)).astype(np.float32)
    xin = x.copy()
    draws = rng.normal(size=(101, S, 9)).astype(np.float32)  # every slot filled: any noise added would show
    trail = np.full((101, S, 9), 7.0, np.float32)
    eps, x0, mean = (np.zeros((S, 9), np.float32) for _ in range(3))
    arr = (C.c_void_p * len(tensors))(*[t.ctypes.data for t in tensors])
    P = lambda a: a.ctypes.data_as(C.c_void_p)
    rc = emu.denoiser_emu_run(arr, P(table), B, N, v, v, g, P(x), P(z), P(draws), P(trail), P(eps), P(x0), P(mean), 3, 20)
    assert rc == 0
    np.testing.assert_array_equal(x, mean)  # the mean itself, no noise
    assert (trail == 7.0).all()  # no trail slot written
    coefs = {"a": float(row[0]), "b": float(row[1]), "c1": float(row[2]), "c2": float(row[3]), "sigma": float(row[4])}
    net = po.build_denoiser(state)
    want, want_x0 = dd.ddim_step(net, torch.from_numpy(xin).reshape(B, N, 9), v, torch.from_numpy(z).reshape(B, N, 384), coefs, None)
    want, want_x0 = want.reshape(S, 9).numpy(), want_x0.reshape(S, 9).numpy()
    np.testing.assert_allclose(x, want, rtol=0, atol=2e-5 * np.abs(want).max() + 1e-5)
    np.testing.assert_allclose(x0, want_x0, rtol=0, atol=1e-5 * np.abs(want_x0).max() + 3e-5 * float(row[1]))
