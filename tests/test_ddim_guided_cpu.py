"""Guided DDIM jumps without a GPU (DESIGN.md "Fewer-step sampling"): the guided-tail rows of pdb_ddim_table_guided against their
float64 formulas, g' = g as today's DDPM tail, the jump times from C and Python, pdb_ddim_table's output unchanged, and the
refusals of the library and of the Python entry points."""
import ctypes as C
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import ddim_guided_oracle as gd
from posediffusion_b200 import _native

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "ddim_table_sha256.json")
GRID = [(1, 2, 1), (1, 10, 1), (1, 10, 3), (7, 10, 5), (10, 10, 2), (3, 10, 9), (45, 10, 7), (20, 30, 4), (40, 60, 13), (1, 99, 50),
        (1, 99, 98), (90, 10, 6)]  # (k, g, g' < g)


def ulps(a, b):
    a, b = np.float32(a), np.float32(b)
    return abs(int(np.array(a).view(np.int32)) - int(np.array(b).view(np.int32))) if np.sign(a) == np.sign(b) or a == b else 1 << 30


@pytest.mark.parametrize("k,g,gs", GRID)
@pytest.mark.parametrize("eta", [0.0, 0.5, 1.0])
def test_guided_rows_match_float64_formulas(k, g, gs, eta):
    t, coef = _native.ddim_table(k + gs, g, eta, guided_steps=gs)
    sched = _native.schedule_table()
    jumps = gd.guided_jumps(g, gs, eta)
    assert jumps[0][0] == g - 1 and jumps[-1][1] == -1
    for i, (want_t, want_s, c) in enumerate(jumps):
        row = coef[k + i]
        assert t[k + i] == want_t and row[5] == want_s
        assert row[0] == sched[want_t, 0] and row[1] == sched[want_t, 1]  # a_t, b_t: the schedule's own values
        for j, name in ((2, "c1"), (3, "c2"), (4, "sigma")):
            assert ulps(row[j], np.float32(c[name])) <= 1, (i, name, row[j], c[name])
    assert (coef[-1, 2], coef[-1, 3], coef[-1, 4]) == (1.0, 0.0, 0.0)  # the last jump lands on x0
    # the prefix is the one the DDPM tail would follow
    t_ddpm, coef_ddpm = _native.ddim_table(k + g, g, eta)
    np.testing.assert_array_equal(t[:k], t_ddpm[:k])
    np.testing.assert_array_equal(coef[:k], coef_ddpm[:k])


@pytest.mark.parametrize("g", [1, 2, 10, 60, 99])
def test_full_guided_steps_is_the_ddpm_tail(g):
    """g' = g: the table holds today's DDPM rows (pdb_ddim_table's output), and at eta = 1 the float64 DDIM jump formulas give those
    rows back -- a_t, b_t exactly, c1 and c2 within 1 ulp."""
    t, coef = _native.ddim_table(1 + g, g, 1.0, guided_steps=g)
    t_ref, coef_ref = _native.ddim_table(1 + g, g, 1.0)
    np.testing.assert_array_equal(t, t_ref)
    np.testing.assert_array_equal(coef, coef_ref)
    sched = _native.schedule_table()
    for i, (ti, si, c) in enumerate(gd.guided_jumps(g, g, 1.0)):
        assert ti == g - 1 - i and si == ti - 1
        assert np.float32(c["a"]) == sched[ti, 0] and np.float32(c["b"]) == sched[ti, 1]
        assert ulps(np.float32(c["c1"]), sched[ti, 2]) <= 1 and ulps(np.float32(c["c2"]), sched[ti, 3]) <= 1, ti


def test_guided_times_from_c_and_python():
    """tau' from the library's table, the binding's helper and the oracle agree for every 1 <= g' <= g <= 99; at g = 100 no
    table exists (the prefix needs k >= 1 <= 100 - g), and the two Python forms still agree."""
    for g in range(1, 101):
        for gs in range(1, g + 1):
            tau = gd.guided_times(g, gs)
            assert _native.guided_times(g, gs) == tau
            assert tau[0] == -1 and tau[-1] == g - 1 and all(b > a for a, b in zip(tau, tau[1:]))
            if g == 100:
                with pytest.raises(ValueError):
                    _native.ddim_table(1 + gs, g, 0.0, guided_steps=gs)
                continue
            t, coef = _native.ddim_table(1 + gs, g, 0.0, guided_steps=gs)
            if gs < g:
                np.testing.assert_array_equal(t[1:], tau[:0:-1])
                np.testing.assert_array_equal(coef[1:, 5], tau[-2::-1])
            else:
                np.testing.assert_array_equal(t[1:], np.arange(g - 1, -1, -1))


def test_ddim_table_output_unchanged():
    """pdb_ddim_table against SHA-256 digests of what it wrote before the guided tail existed (tests/golden), refusals included."""
    lib = _native.load_library()
    cases = json.load(open(GOLDEN))["cases"]
    assert len(cases) > 100
    for case in cases:
        steps = case["steps"]
        t = np.zeros(128, np.int32)
        coef = np.zeros((128, 8), np.float32)
        rc = lib.pdb_ddim_table(steps, case["guide_below"], case["eta"], 1e-4, 0.1, t.ctypes.data_as(C.c_void_p),
                                coef.ctypes.data_as(C.c_void_p))
        assert rc == case["rc"], case
        if rc == 0:
            assert hashlib.sha256(t[:steps].tobytes() + coef[:steps].tobytes()).hexdigest() == case["sha256"], case


@pytest.mark.parametrize("steps,g,gs,eta", [(5, 10, 0, 0.0), (15, 10, 11, 0.0), (5, 0, 1, 0.0), (5, 10, -1, 0.0), (5, 10, 5, 0.0),
                                            (96, 10, 5, 0.0), (101, 10, 10, 0.0), (6, 100, 5, 0.0), (10, 10, 5, -0.1),
                                            (10, 10, 5, float("nan")), (10, 10, 5, float("inf")), (10, 10, 5, 50.0)])
def test_invalid_arguments_refused(steps, g, gs, eta):
    lib = _native.load_library()
    t = np.zeros(128, np.int32)
    coef = np.zeros((128, 8), np.float32)
    rc = lib.pdb_ddim_table_guided(steps, g, gs, eta, 1e-4, 0.1, t.ctypes.data_as(C.c_void_p), coef.ctypes.data_as(C.c_void_p))
    assert rc == -1  # PDB_ERR_INVALID
    with pytest.raises(ValueError):
        _native.ddim_table(steps, g, eta, guided_steps=gs)
    if eta != 50.0:  # 1 - abar_s - sigma^2 < 0 is the library's check alone, as for the prefix
        with pytest.raises(ValueError):
            _native.ddim_check(steps, g, eta, gs)


def test_null_outputs_refused():
    assert _native.load_library().pdb_ddim_table_guided(10, 10, 5, 0.0, 1e-4, 0.1, None, None) == -1


def test_python_check():
    assert _native.ddim_check(15, 10, 0.0, 5) == 10
    assert _native.ddim_check(11, 10, 0.0, 1) == 10
    assert _native.ddim_check(20, 10, 0.0, 10) == _native.ddim_check(20, 10, 0.0) == 10
    assert _native.ddim_check(95, 10, 1.0, 5) == 90  # k = 100 - g with a shorter tail
    for steps, g, gs in ((15, 0, 5), (15, 10, 0), (25, 10, 11), (5, 10, 5), (96, 10, 5)):
        with pytest.raises(ValueError):
            _native.ddim_check(steps, g, 0.0, gs)


def _model():
    import posediffusion_b200 as pdb

    return pdb.PoseDiffusionModel(
        pose_encoding_type="absT_quaR_logFL", IMAGE_FEATURE_EXTRACTOR=None,
        DIFFUSER={"_target_": "models.GaussianDiffusion", "beta_schedule": "custom"},
        DENOISER={"_target_": "models.Denoiser", "TRANSFORMER": dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8,
                                                                     dropout=0.1, batch_first=True, norm_first=True,
                                                                     _target_="models.TransformerEncoderWrapper")},
    )


def test_python_argument_validation():
    model = _model()
    dif = model.diffuser
    z = torch.zeros(1, 5, 384)
    for kw in (dict(sampling_timesteps=15, guided_steps=5),  # no cond_fn
               dict(sampling_timesteps=15, cond_fn=print, cond_start_step=0, guided_steps=5),
               dict(sampling_timesteps=15, cond_fn=print, cond_start_step=10, guided_steps=0),
               dict(sampling_timesteps=25, cond_fn=print, cond_start_step=10, guided_steps=11),
               dict(sampling_timesteps=5, cond_fn=print, cond_start_step=10, guided_steps=5),
               dict(sampling_timesteps=96, cond_fn=print, cond_start_step=10, guided_steps=5)):
        with pytest.raises(ValueError):
            dif.ddim_sample([1, 5, 9], z, **kw)
    with pytest.raises(ValueError, match="sampling_timesteps"):
        model(z=z, training=False, guided_steps=5, cond_fn=print, cond_start_step=10)
