"""Every sampling-loop entry point refuses a bad call before it enqueues anything: the expected return code (or, where the binding
checks first, exception), no launch, the pose buffer untouched, and the next good call on the same context succeeds.

The C entries are called directly, so that each refusal is the library's own and not the binding's.  Every buffer is sized for a
129-frame call, so a call that were not refused could not write past it."""
import ctypes as C

import numpy as np
import pytest
import torch

from conftest import load_golden

import posediffusion_b200 as pdb
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn

pytestmark = pytest.mark.gpu
TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
N, G, K, GS, ETA = 5, 10, 10, 5, 0.5  # frames, guided timesteps, DDIM prefix steps, guided DDIM jumps, eta
MAXF = _native.MAX_FRAMES + 1  # buffers hold a call of this many frames (batch 1) or of 2 x N frames
SENTINEL = 1234.5
INVALID, STATE, LIMIT = _native.PDB_ERR_INVALID, _native.PDB_ERR_STATE, _native.PDB_ERR_LIMIT

DEVICE = ("pdb_sample_loop", "pdb_sample_loop_ddim", "pdb_sample_loop_ddim_guided")
HOST = ("pdb_sample_loop_host", "pdb_sample_loop_host_matches", "pdb_sample_loop_host_matches_ddim")
DDIM = ("pdb_sample_loop_ddim", "pdb_sample_loop_ddim_guided", "pdb_sample_loop_host_matches_ddim")
MATCH_ARRAYS = ("pdb_sample_loop_host_matches", "pdb_sample_loop_host_matches_ddim")

# (case, argument changes, expected return code)
CASES = [
    ("null_z", dict(z=None), INVALID),
    ("null_draws", dict(draws=None), INVALID),
    ("null_pose", dict(pose=None), INVALID),  # the pose buffer still holds the sentinel: the call had no pointer to it
    ("batch_0", dict(batch=0, n_problems=0), INVALID),
    ("frames_129", dict(frames=_native.MAX_FRAMES + 1, problems=None), LIMIT),  # no sets: they would be refused for their frames
    ("n_problems", dict(batch=2), INVALID),
    ("cfg_null", dict(cfg=None), INVALID),
    ("other_frame_count", dict(problems="six"), INVALID),
    ("iter_num", dict(cfg="iter_num"), INVALID),
    ("no_weights", dict(ctx="unloaded"), STATE),
    ("k_0", dict(k=0), INVALID),
    ("k_too_large", dict(k=_native.NUM_TIMESTEPS - G + 1), INVALID),
    ("guided_steps_0", dict(gs=0), INVALID),
    ("guided_steps_above_g", dict(gs=G + 1), INVALID),
    ("eta_negative", dict(eta=-0.5), INVALID),
    ("eta_nan", dict(eta=float("nan")), INVALID),
    ("eta_too_large", dict(eta=50.0), INVALID),  # 1 - abar_s - sigma^2 < 0
]


def applies(entry, case):
    if case.startswith(("k_", "eta_")):
        return entry in DDIM
    if case.startswith("guided_steps_"):
        return entry in DDIM and entry != "pdb_sample_loop_ddim"  # whose g' is g
    if case in ("n_problems", "other_frame_count"):
        return entry not in MATCH_ARRAYS  # the host arrays carry neither: the binding refuses them (last test)
    return True


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need an H100"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def den(dev):
    g = load_golden("denoiser.npz")
    d = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    d.load_state_dict(syn.random_denoiser_state(int(g["weight_seed"]), float(g["bias_std"])), strict=True)
    return d.to(dev)


@pytest.fixture(scope="module")
def setup(den, dev):
    ctx = den.native_context()
    scene = syn.scene_matches(N, 32, seed=5)[0]
    cfg = dict(syn.default_ggs_cfg(), iter_num=2, min_matches=1e9, verbose=False)  # every GGS phase dropped: a finite pose
    z = np.zeros(MAXF * _native.Z_DIM, np.float32)
    z[: N * _native.Z_DIM] = syn.random_features(1, N, 5).numpy().ravel()
    draws = np.zeros((_native.NUM_TIMESTEPS + 1) * MAXF * 9, np.float32)
    draws[: (_native.NUM_TIMESTEPS + 1) * N * 9] = syn.predraw_noise(1, N, seed=5).numpy().ravel()
    return dict(ctx=ctx, scene=scene, cfg=cfg, z=z, draws=draws, z_dev=torch.from_numpy(z).to(dev),
                draws_dev=torch.from_numpy(draws).to(dev), sets={N: [ctx.pack_matches(scene)],
                                                                  "six": [ctx.pack_matches(syn.scene_matches(6, 32, seed=6)[0])]},
                stream=C.c_void_p(torch.cuda.current_stream(dev).cuda_stream))


def call(s, entry, ctx, pose, batch=1, frames=N, z=True, draws=True, problems=N, cfg="good", k=K, gs=None, eta=ETA, n_problems=1):
    """The C entry `entry` on `ctx` with the good call's arguments (pose: the output buffer), changed as the case asks."""
    host = entry in HOST
    zp = None if z is None else (s["z"].ctypes.data if host else s["z_dev"].data_ptr())
    dp = None if draws is None else (s["draws"].ctypes.data if host else s["draws_dev"].data_ptr())
    pp = None if pose is None else (pose.ctypes.data if host else pose.data_ptr())
    conf = None
    if cfg is not None:
        conf = _native.ggs_config_struct(dict(s["cfg"], iter_num=-1) if cfg == "iter_num" else s["cfg"])
    conf = C.byref(conf) if conf is not None else None
    gs = (G if entry == "pdb_sample_loop_ddim" else GS) if gs is None else gs
    ddim = (k + gs, eta) + ((gs,) if entry != "pdb_sample_loop_ddim" else ())
    head = (ctx.handle, zp, dp, batch, frames) + (ddim if entry in DDIM else ())
    tail = (conf, G, pp, None, None, s["stream"])
    if entry in MATCH_ARRAYS:
        ptrs, counts, _, _keep = ctx._host_match_arrays([s["scene"]], 1, N)
        height, width = (int(v) for v in s["scene"]["img_shape"][2:])
        with torch.cuda.device(ctx.device):
            return getattr(ctx.lib, entry)(*head, ptrs[0], ptrs[1], ptrs[2], counts, height, width, *tail)
    arr = ctx._problem_array(s["sets"][problems]) if problems is not None else None
    with torch.cuda.device(ctx.device):
        return getattr(ctx.lib, entry)(*head, arr, n_problems if problems is not None else 0, *tail)


@pytest.mark.parametrize("entry,case,change,rc",
                         [pytest.param(e, *c, id=f"{e}-{c[0]}") for e in DEVICE + HOST for c in CASES if applies(e, c[0])])
def test_refused_before_anything_is_enqueued(setup, den, dev, entry, case, change, rc):
    s = setup
    ctx = s["ctx"]
    owned = None
    if change.get("ctx") == "unloaded":
        ctx = owned = _native.Context(dev.index)  # a second context on the same device, no weights loaded
    kw = {k: v for k, v in change.items() if k != "ctx"}
    host = entry in HOST
    pose = np.full(MAXF * 9, SENTINEL, np.float32) if host else torch.full((MAXF * 9,), SENTINEL, device=dev)
    try:
        torch.cuda.synchronize()
        before = ctx.launch_count
        got = call(s, entry, ctx, kw.pop("pose", pose), **kw)
        assert got == rc, (got, ctx.lib.pdb_last_error(ctx.handle))
        torch.cuda.synchronize()
        assert ctx.launch_count == before
        assert (pose == SENTINEL).all()
        if owned is not None:
            ctx.load_denoiser(den.ordered_parameters())
        assert call(s, entry, ctx, pose) == 0, ctx.lib.pdb_last_error(ctx.handle)
        torch.cuda.synchronize()
        first = pose[: N * 9]
        assert bool(np.isfinite(first).all() if host else torch.isfinite(first).all()) and (first != SENTINEL).all()
    finally:
        if owned is not None:
            torch.cuda.synchronize()
            owned.lib.pdb_destroy(owned.handle)


@pytest.mark.parametrize("ddim", [False, True], ids=["ddpm", "ddim"])
def test_host_matches_binding_refusals(setup, dev, ddim):
    """The match-array entries take one set per sequence and no frame count of their own: the binding refuses a count or frame
    count that does not fit, before the library is called."""
    s = setup
    ctx = s["ctx"]
    slots = (1 + K if ddim else _native.NUM_TIMESTEPS + 1)
    z2 = np.ascontiguousarray(np.concatenate([s["z"][: N * 384]] * 2).reshape(2, N, 384))
    d2 = np.ascontiguousarray(np.repeat(s["draws"][: slots * N * 9].reshape(slots, 1, N, 9), 2, axis=1))
    z1, d1 = z2[:1].copy(), np.ascontiguousarray(d2[:, :1])
    six = syn.scene_matches(6, 32, seed=6)[0]
    extra = (G, K + GS, ETA) if ddim else (G,)
    kw = dict(guided_steps=GS) if ddim else {}
    run = ctx.sample_loop_host_matches_ddim if ddim else ctx.sample_loop_host_matches
    torch.cuda.synchronize()
    before = ctx.launch_count
    pose2, pose1 = np.full((2, N, 9), SENTINEL, np.float32), np.full((1, N, 9), SENTINEL, np.float32)
    with pytest.raises(ValueError, match="one per sequence"):
        run(z2, d2, [s["scene"]], s["cfg"], *extra, pose2, **kw)
    with pytest.raises(ValueError, match="6 frames used with 5"):
        run(z1, d1, [six], s["cfg"], *extra, pose1, **kw)
    torch.cuda.synchronize()
    assert ctx.launch_count == before and (pose2 == SENTINEL).all() and (pose1 == SENTINEL).all()
    run(z1, d1, [s["scene"]], s["cfg"], *extra, pose1, **kw)
    assert np.isfinite(pose1).all() and (pose1 != SENTINEL).all()
