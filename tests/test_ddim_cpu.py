"""DDIM step tables and argument checks without a GPU: pdb_ddim_table against its float64 formulas (DESIGN.md "Fewer-step
sampling"), DDPM as its special case (k = 100 - g, eta = 1), the refusals, and the oracle's DDIM loop against the oracle's DDPM
loop in float64."""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import ddim_oracle as dd
from oracle.denoiser_f64 import DenoiserF64
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

GRID = [(1, 0), (1, 10), (1, 99), (3, 0), (3, 10), (7, 10), (10, 0), (20, 10), (33, 5), (45, 10), (90, 10), (99, 1), (100, 0)]


def ulps(a, b):
    a, b = np.float32(a), np.float32(b)
    return abs(int(np.array(a).view(np.int32)) - int(np.array(b).view(np.int32))) if np.sign(a) == np.sign(b) or a == b else 1 << 30


@pytest.mark.parametrize("k,g", GRID)
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_table_matches_float64_formulas(k, g, eta):
    t, coef = _native.ddim_table(k + g, g, eta)
    tau = dd.ddim_times(k, g)
    assert tau[-1] == 99 and tau[0] == g - 1
    abar = dd.alphas_cumprod_f64()
    sched = _native.schedule_table()
    for i in range(k):
        want_t, want_s = tau[k - i], tau[k - i - 1]
        assert t[i] == want_t
        c = dd.ddim_coef_f64(want_t, want_s, eta, abar)
        row = coef[i]
        assert row[0] == sched[want_t, 0] and row[1] == sched[want_t, 1]  # a_t, b_t: the schedule's own values
        for j, name in ((2, "c1"), (3, "c2"), (4, "sigma")):
            assert ulps(row[j], np.float32(c[name])) <= 1, (i, name, row[j], c[name])
        assert row[5] == want_s
        if eta == 0.0:
            assert row[4] == 0.0
        if want_s == -1:
            assert (row[2], row[3], row[4]) == (1.0, 0.0, 0.0)
    for i in range(g):  # the guided tail: DDPM rows of t = g-1 .. 0
        assert t[k + i] == g - 1 - i
        np.testing.assert_array_equal(coef[k + i], sched[g - 1 - i])


def test_single_jump_lands_on_the_hand_over():
    for g in (0, 1, 10, 50):
        t, coef = _native.ddim_table(1 + g, g, 0.0)
        assert t[0] == 99 and coef[0, 5] == g - 1


@pytest.mark.parametrize("g", [0, 1, 10, 60])
def test_full_steps_eta_one_is_ddpm(g):
    """k = 100 - g visits every timestep; with eta = 1 each row is the DDPM posterior row: c1 and c2 within 1 ulp, sigma within
    2e-7 relative (DDPM stores exp(0.5 * float32 log variance)).  At t = 0 DDPM stores the clamped 1e-10 and the DDIM row 0;
    neither sampler adds noise at that step."""
    k = 100 - g
    t, coef = _native.ddim_table(k + g, g, 1.0)
    sched = _native.schedule_table()
    np.testing.assert_array_equal(t[:k], np.arange(99, g - 1, -1))
    for i in range(k):
        ti = int(t[i])
        assert ulps(coef[i, 2], sched[ti, 2]) <= 1 and ulps(coef[i, 3], sched[ti, 3]) <= 1, ti
        if ti == 0:
            assert coef[i, 4] == 0.0 and abs(sched[ti, 4] - 1e-10) < 1e-15
        else:
            assert abs(float(coef[i, 4]) / float(sched[ti, 4]) - 1.0) <= 2e-7, ti


@pytest.mark.parametrize("steps,g,eta", [(0, 0, 0.0), (10, 10, 0.0), (101, 0, 0.0), (101, 10, 0.0), (5, -1, 0.0), (5, 101, 0.0),
                                         (10, 0, -0.1), (10, 0, float("nan")), (10, 0, float("inf")), (10, 0, 50.0)])
def test_invalid_arguments_refused(steps, g, eta):
    lib = _native.load_library()
    t = np.zeros(128, np.int32)
    coef = np.zeros((128, 8), np.float32)
    rc = lib.pdb_ddim_table(steps, g, eta, 1e-4, 0.1, t.ctypes.data_as(C.c_void_p), coef.ctypes.data_as(C.c_void_p))
    assert rc == -1  # PDB_ERR_INVALID
    with pytest.raises(ValueError):
        _native.ddim_table(steps, g, eta)


def test_null_outputs_refused():
    assert _native.load_library().pdb_ddim_table(10, 0, 0.0, 1e-4, 0.1, None, None) == -1


def test_step_times_integer_arithmetic():
    for g in range(0, 100, 7):
        for k in range(1, 101 - g):
            tau = dd.ddim_times(k, g)
            assert tau[0] == g - 1 and tau[-1] == 99
            assert all(b > a for a, b in zip(tau, tau[1:]))  # strictly decreasing in the order they run
            t, _ = _native.ddim_table(k + g, g, 0.0)
            np.testing.assert_array_equal(t[:k], tau[:0:-1])


def test_oracle_ddim_full_steps_eta_one_equals_ddpm_f64():
    """The oracle's DDIM at k = 100 and eta = 1 is the oracle's DDPM loop in float64: from the same state, network output and draw,
    every one of the 100 updates agrees to 1e-12 (the loop itself is chaotic, so the comparison is per step)."""
    torch.manual_seed(0)
    net = DenoiserF64(syn.random_denoiser_state(3, 0.05)).net64
    B, N = 1, 3
    z = syn.random_features(B, N, 5).double()
    draws = torch.randn(101, B, N, 9, dtype=torch.float64)
    beta = torch.linspace(1e-4, 0.1, 100, dtype=torch.float64)
    abar = torch.cumprod(1 - beta, 0)
    abar_prev = torch.cat([torch.ones(1, dtype=torch.float64), abar[:-1]])
    steps = dd.prefix_steps(100, 0, 1.0)
    x = draws[0].clone()
    with torch.no_grad():
        for i, t in enumerate(reversed(range(100))):
            eps = net(x, torch.full((B,), t, dtype=torch.long), z)
            x0 = (1 / abar[t]).sqrt() * x - (1 / abar[t] - 1).sqrt() * eps
            mean = beta[t] * abar_prev[t].sqrt() / (1 - abar[t]) * x0 + (1 - abar_prev[t]) * (1 - beta[t]).sqrt() / (1 - abar[t]) * x
            var = beta[t] * (1 - abar_prev[t]) / (1 - abar[t])
            ddpm = mean + var.sqrt() * draws[1 + i] if t > 0 else mean
            ts, _s, c = steps[i]
            assert ts == t
            ddim = c["c1"] * (c["a"] * x - c["b"] * eps) + c["c2"] * x + c["sigma"] * draws[1 + i]
            assert (ddim - ddpm).abs().max().item() <= 1e-12 * max(1.0, ddpm.abs().max().item()), t
            x = ddpm


def test_python_argument_validation():
    import posediffusion_b200 as pdb

    dif = pdb.GaussianDiffusion()
    dif.model = pdb.Denoiser(TRANSFORMER=dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1,
                                              batch_first=True, norm_first=True))
    z = torch.zeros(1, 5, 384)
    for kw in (dict(sampling_timesteps=0), dict(sampling_timesteps=101), dict(sampling_timesteps=10, eta=-1.0),
               dict(sampling_timesteps=10, eta=float("nan")), dict(sampling_timesteps=10, cond_fn=print, cond_start_step=10),
               dict(sampling_timesteps=50, cond_fn=print, cond_start_step=60)):
        with pytest.raises(ValueError):
            dif.ddim_sample([1, 5, 9], z, **kw)
    assert _native.ddim_check(20, 10, 0.0) == 10
    assert _native.ddim_check(100, 0, 1.0) == 100
    with pytest.raises(ValueError):
        _native.ddim_check(20, 0, math.inf)
