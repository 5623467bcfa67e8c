"""ctypes binding of libposediff_b200.so (include/posediff_b200.h).

PyTorch is used here only for device memory and streams.  There is NO fallback: if the library is
missing, or no sm_90 GPU is present, every compute call raises.
"""
from __future__ import annotations

import ctypes as C
import itertools
import math
import os
import threading
from typing import Dict, List, Optional, Sequence

import numpy as np
import torch

_PKG = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_PKG, "libposediff_b200.so")

PDB_NUM_WEIGHT_TENSORS = 108
PDB_GGS_PHASES = 5
NUM_TIMESTEPS = 100
TARGET_DIM = 9
Z_DIM = 384
MAX_FRAMES = 128
PDB_VIT_NUM_TENSORS = 150
VIT_DIM = 384


class NativeError(RuntimeError):
    pass


class GgsConfig(C.Structure):
    _fields_ = [
        ("alpha", C.c_double),
        ("learning_rate", C.c_double),
        ("iter_num", C.c_int32),
        ("sampson_max", C.c_double),
        ("min_matches", C.c_double),
        ("momentum", C.c_double),
    ]


class GgsStats(C.Structure):
    _fields_ = [
        ("sampson", C.c_float * PDB_GGS_PHASES),
        ("iters", C.c_int32 * PDB_GGS_PHASES),
        ("dropped", C.c_int32 * PDB_GGS_PHASES),
        ("n_valid", C.c_int32 * PDB_GGS_PHASES),
    ]


GGS_STATS_DTYPE = np.dtype(
    [("sampson", np.float32, (PDB_GGS_PHASES,)), ("iters", np.int32, (PDB_GGS_PHASES,)),
     ("dropped", np.int32, (PDB_GGS_PHASES,)), ("n_valid", np.int32, (PDB_GGS_PHASES,))]
)
assert GGS_STATS_DTYPE.itemsize == C.sizeof(GgsStats)

EXPORTS = {
    # name: (restype, argtypes)
    "pdb_abi_version": (C.c_int, []),
    "pdb_create": (C.c_int, [C.POINTER(C.c_void_p), C.c_int]),
    "pdb_destroy": (None, [C.c_void_p]),
    "pdb_last_error": (C.c_char_p, [C.c_void_p]),
    "pdb_device_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "pdb_launch_count": (C.c_int64, [C.c_void_p]),
    "pdb_profile_enable": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdb_profile_read": (C.c_int, [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int64), C.POINTER(C.c_double), C.POINTER(C.c_int64)]),
    "pdb_debug_ggs_clocks": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_int32]),
    "pdb_denoiser_engine": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdb_debug_tc_linear": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]),
    "pdb_schedule_table": (C.c_int, [C.c_void_p, C.c_double, C.c_double]),
    "pdb_ddim_table": (C.c_int, [C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p]),
    "pdb_sample_loop_ddim": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.POINTER(C.c_void_p),
                                       C.c_int32, C.POINTER(GgsConfig), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_ddim_table_guided": (C.c_int, [C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p]),
    "pdb_sample_loop_ddim_guided": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32,
                                              C.POINTER(C.c_void_p), C.c_int32, C.POINTER(GgsConfig), C.c_int32, C.c_void_p, C.c_void_p,
                                              C.c_void_p, C.c_void_p]),
    "pdb_sample_loop_host_matches_ddim": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_int32,
                                                    C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int64),
                                                    C.c_int32, C.c_int32, C.POINTER(GgsConfig), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p]),
    "pdb_denoiser_load": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p]),
    "pdb_denoiser_forward": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p]),
    "pdb_p_sample": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_matches_pack": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "pdb_matches_pack_colmap": (C.c_int, [C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p,
                                          C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.POINTER(C.c_void_p)]),
    "pdb_matches_free": (None, [C.c_void_p]),
    "pdb_matches_info": (C.c_int, [C.c_void_p, C.POINTER(C.c_int64), C.POINTER(C.c_int32), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "pdb_debug_tc_swap": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdb_debug_denoiser_handover": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdb_ggs_layout": (C.c_int, [C.c_void_p, C.c_int32]),
    "pdb_ggs_layout_get": (C.c_int, [C.c_void_p]),
    "pdb_debug_pack_layout": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64, C.c_int32, C.c_int32, C.c_void_p, C.c_int32,
                                        C.c_void_p, C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int64)]),
    "pdb_sampson_eval": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_ggs": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_int32, C.c_void_p, C.POINTER(GgsConfig), C.c_void_p, C.c_void_p]),
    "pdb_sample_loop": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.c_int32, C.POINTER(GgsConfig), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_pose_to_camera": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_rel_pose_error": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_cameras_align": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_double,
                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_vit_load": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.c_int32, C.c_void_p]),
    "pdb_vit_pos_table": (C.c_int, [C.c_void_p, C.c_int32, C.c_int32, C.c_void_p]),
    "pdb_extract_features": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_double), C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p]),
    "pdb_extract_features_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_double), C.c_int32, C.c_void_p, C.c_void_p]),
    "pdb_sample_loop_host": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.c_int32, C.POINTER(GgsConfig), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_sample_loop_host_matches": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_int64), C.c_int32, C.c_int32, C.POINTER(GgsConfig), C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_images_preprocess_host": (C.c_int, [C.c_void_p, C.c_int32, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p]),
    "pdb_train_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32]),
    "pdb_train_forward": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                    C.c_float, C.c_uint64, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_train_backward": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p]),
    "pdb_train_backward_z": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p,
                                       C.c_void_p]),
    "pdb_vit_train_workspace_bytes": (C.c_int64, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_double), C.c_int32]),
    "pdb_vit_train_forward": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_double),
                                        C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p]),
    "pdb_vit_backward": (C.c_int, [C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p]),
    "pdb_camera_to_pose": (C.c_int, [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_double, C.c_double, C.c_double,
                                     C.c_void_p, C.c_void_p]),
    "pdb_dropout_mask_host": (C.c_int, [C.c_uint64, C.c_int32, C.c_int32, C.c_int64, C.c_int64, C.c_float, C.c_void_p]),
}

TRAIN_MAX_FRAMES = 64
LOSS_TYPES = {"l1": 0, "l2": 1}
DROPOUT_SITES = {"attn": 0, "out_proj": 1, "relu": 2, "linear2": 3}


def dropout_mask_host(seed: int, layer: int, site: int, offset: int, count: int, p: float) -> np.ndarray:
    """Keep mask (uint8, 1 = kept) of `count` elements from `offset` of dropout site `site` of layer `layer`: the same Philox
    function the training kernels evaluate (no GPU needed)."""
    out = np.zeros(max(int(count), 0), dtype=np.uint8)
    rc = load_library().pdb_dropout_mask_host(int(seed) & (2**64 - 1), int(layer), int(site), int(offset), int(count), float(p),
                                              out.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise ValueError(f"pdb_dropout_mask_host rejected (layer={layer}, site={site}, offset={offset}, count={count}, p={p})")
    return out


def train_workspace_bytes(batch: int, frames: int) -> int:
    return int(load_library().pdb_train_workspace_bytes(int(batch), int(frames)))


def vit_train_workspace_bytes(n_images: int, height: int, width: int, scale_factors: Sequence[float]) -> int:
    """Bytes of the workspace a backbone training forward of this shape needs; 0 for an unsupported shape (no GPU needed)."""
    sf = (C.c_double * max(len(scale_factors), 1))(*[float(f) for f in scale_factors])
    return int(load_library().pdb_vit_train_workspace_bytes(int(n_images), int(height), int(width), sf, len(scale_factors)))


_lib = None
_lib_lock = threading.Lock()


def load_library() -> C.CDLL:
    """dlopen the in-tree library and bind every symbol the header declares."""
    global _lib
    with _lib_lock:
        if _lib is None:
            if not os.path.exists(LIB_PATH):
                raise NativeError(
                    f"{LIB_PATH} is missing: build it with `python -m posediffusion_b200.build` "
                    "(posediffusion_b200 has no CPU or PyTorch fallback)"
                )
            lib = C.CDLL(LIB_PATH)
            for name, (res, args) in EXPORTS.items():
                fn = getattr(lib, name)  # AttributeError if the symbol is not exported
                fn.restype = res
                fn.argtypes = args
            if lib.pdb_abi_version() != PDB_ABI_VERSION:
                raise NativeError(f"{LIB_PATH} has ABI version {lib.pdb_abi_version()}, this binding expects {PDB_ABI_VERSION}: "
                                  "rebuild with `python -m posediffusion_b200.build --force`")
            _lib = lib
    return _lib


def schedule_table(beta_1: float = 1e-4, beta_T: float = 0.1) -> np.ndarray:
    """[100, 8] float32 DDPM coefficients from the library's host helper (no GPU needed)."""
    out = np.zeros((NUM_TIMESTEPS, 8), dtype=np.float32)
    rc = load_library().pdb_schedule_table(out.ctypes.data_as(C.c_void_p), beta_1, beta_T)
    if rc != 0:
        raise NativeError(f"pdb_schedule_table failed ({rc})")
    return out


def ddim_table(steps: int, guide_below: int = 0, eta: float = 0.0, beta_1: float = 1e-4, beta_T: float = 0.1,
               guided_steps: Optional[int] = None):
    """(t [steps] int32, coef [steps, 8] float32): the DDIM step table of pdb_ddim_table_guided -- `steps` denoiser evaluations,
    the last g' = `guided_steps` (default `guide_below`) of them the guided tail over timesteps guide_below-1 .. 0: DDPM rows when
    g' = guide_below, DDIM jumps when g' is smaller (no GPU needed).  ValueError where the library refuses the arguments."""
    gs = int(guide_below) if guided_steps is None else int(guided_steps)
    n = max(int(steps), 1)
    t = np.zeros(n, dtype=np.int32)
    coef = np.zeros((n, 8), dtype=np.float32)
    rc = load_library().pdb_ddim_table_guided(int(steps), int(guide_below), gs, float(eta), beta_1, beta_T,
                                              t.ctypes.data_as(C.c_void_p), coef.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise ValueError(f"pdb_ddim_table_guided refused steps={steps}, guide_below={guide_below}, guided_steps={gs}, eta={eta}")
    return t, coef


def guided_times(g: int, guided_steps: int) -> List[int]:
    """tau'_0 .. tau'_{g'} = floor(j g / g') - 1 of the g' guided jumps over timesteps g-1 .. 0 (pdb_ddim_table_guided); jump i
    runs the network at tau'_{g'-i}."""
    return [(j * int(g)) // int(guided_steps) - 1 for j in range(int(guided_steps) + 1)]


def clamp_guided(cond_start_step: int) -> int:
    """g = clamp(cond_start_step, 0, 100): the timesteps a sampling loop guides."""
    return max(0, min(int(cond_start_step), NUM_TIMESTEPS))


def ddim_check(steps: int, guided: int, eta: float, guided_steps: Optional[int] = None) -> int:
    """k = steps - g' unguided DDIM steps (g' = `guided_steps`, default `guided`), or ValueError (the library's own check, mirrored
    so that nothing is enqueued)."""
    g = int(guided)
    if guided_steps is not None:
        if g == 0:
            raise ValueError(f"guided_steps={guided_steps} without guidance (no cond_fn, or cond_start_step 0)")
        if not 1 <= int(guided_steps) <= g:
            raise ValueError(f"guided_steps={guided_steps}: the {g} guided timesteps take 1 .. {g} denoiser steps")
    gs = g if guided_steps is None else int(guided_steps)
    k = int(steps) - gs
    if not 1 <= k <= NUM_TIMESTEPS - g:
        raise ValueError(f"sampling_timesteps={steps} with {gs} guided steps leaves {k} unguided DDIM steps; "
                         f"1 .. {NUM_TIMESTEPS - g} are possible")
    if not math.isfinite(float(eta)) or float(eta) < 0.0:
        raise ValueError(f"eta={eta}: DDIM needs a finite eta >= 0")
    return k


def vit_pos_table(pos_embed: np.ndarray, grid_h: int, grid_w: int) -> np.ndarray:
    """interpolate_pos_encoding of the DINO backbone for a grid_h x grid_w patch grid (host helper, no GPU needed)."""
    pos = np.ascontiguousarray(pos_embed, dtype=np.float32).reshape(197, VIT_DIM)
    out = np.zeros((1 + grid_h * grid_w, VIT_DIM), dtype=np.float32)
    rc = load_library().pdb_vit_pos_table(pos.ctypes.data_as(C.c_void_p), grid_h, grid_w, out.ctypes.data_as(C.c_void_p))
    if rc != 0:
        raise NativeError(f"pdb_vit_pos_table failed ({rc})")
    return out


_module_tokens = itertools.count(1)


def module_token() -> int:
    """Process-unique, never reused identity of a module for the device-side weight caches (`id()` of a freed module can come
    back for a new one whose parameters land in the same allocator blocks with the same versions)."""
    return next(_module_tokens)


GGS_LAYOUTS = {"plain": 0, "paired": 1}
PDB_ABI_VERSION = 2  # include/posediff_b200.h
PDB_OK, PDB_ERR_INVALID, PDB_ERR_CUDA, PDB_ERR_STATE, PDB_ERR_LIMIT = 0, -1, -2, -3, -4


def pack_layout_host(matches_dict: Dict, layout: str = "plain"):
    """Host image of the packed match stream exactly as pdb_matches_pack lays it out in HBM (no GPU needed; used by the CPU
    tests of the layout contract).  Returns (segs [nseg,4] int32 {first_round, count, a, b}, pts [rounds*32, 4] float32)."""
    frames = int(matches_dict["img_shape"][0])
    kp1 = np.ascontiguousarray(matches_dict["kp1"], dtype=np.float64).reshape(-1, 2)
    kp2 = np.ascontiguousarray(matches_dict["kp2"], dtype=np.float64).reshape(-1, 2)
    i12 = np.ascontiguousarray(matches_dict["i12"], dtype=np.int64).reshape(-1, 2)
    lib = load_library()
    nseg, rounds = C.c_int32(), C.c_int64()
    args = (kp1.ctypes.data, kp2.ctypes.data, i12.ctypes.data, len(kp1), frames, GGS_LAYOUTS[layout])
    rc = lib.pdb_debug_pack_layout(*args, None, 0, None, 0, C.byref(nseg), C.byref(rounds))
    if rc != 0:
        raise ValueError(f"pdb_debug_pack_layout failed ({rc})")
    segs = np.zeros((max(nseg.value, 1), 4), dtype=np.int32)
    pts = np.full((max(rounds.value, 1) * 32, 4), np.nan, dtype=np.float32)
    rc = lib.pdb_debug_pack_layout(*args, segs.ctypes.data, nseg.value, pts.ctypes.data, rounds.value, C.byref(nseg), C.byref(rounds))
    if rc != 0:
        raise ValueError(f"pdb_debug_pack_layout failed ({rc})")
    return segs[: nseg.value], pts[: rounds.value * 32]


def ggs_config_struct(cfg: Dict) -> GgsConfig:
    """cfgs/default.yaml GGS section / kwargs of GGS_optimize -> pdb_ggs_config."""
    enc = cfg.get("pose_encoding_type", "absT_quaR_logFL")
    if enc != "absT_quaR_logFL":
        raise ValueError(f"Unknown pose encoding {enc}")  # camera_transform.py:98-99
    return GgsConfig(
        alpha=float(cfg.get("alpha", 1e-4)),
        learning_rate=float(cfg.get("learning_rate", 1e-2)),
        iter_num=int(cfg.get("iter_num", 100)),
        sampson_max=float(cfg.get("sampson_max", 10)),
        min_matches=float(cfg.get("min_matches", 10)),
        momentum=float(cfg.get("momentum", 0.9)),
    )


def _stream_ptr(device: torch.device) -> C.c_void_p:
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def _check_dev(t: torch.Tensor, name: str, device: torch.device, shape=None):
    if not t.is_cuda:
        raise NativeError(f"{name} must be a CUDA tensor (posediffusion_b200 has no CPU fallback)")
    if t.device != device:
        raise NativeError(f"{name} is on {t.device}, context is on {device}")
    if t.dtype != torch.float32 or not t.is_contiguous():
        raise NativeError(f"{name} must be contiguous float32")
    if shape is not None and tuple(t.shape) != tuple(shape):
        raise NativeError(f"{name} has shape {tuple(t.shape)}, expected {tuple(shape)}")


class Matches:
    """Device-resident packed correspondences of one sequence (pdb_matches)."""

    def __init__(self, ctx: "Context", handle: C.c_void_p, frames: int, m_total: int):
        self.ctx, self.handle, self.frames, self.m_total = ctx, handle, frames, m_total
        info = (C.c_int64(), C.c_int32(), C.c_int64(), C.c_int32())
        ctx.lib.pdb_matches_info(handle, *[C.byref(v) for v in info])
        self.segments, self.rounds = info[1].value, info[2].value

    def __del__(self):
        try:
            if self.handle:
                self.ctx.lib.pdb_matches_free(self.handle)
                self.handle = None
        except Exception:
            pass


class Context:
    """One pdb_context per (process, GPU)."""

    _by_device: Dict[int, "Context"] = {}

    def __init__(self, device_index: int):
        self.lib = load_library()
        self.device = torch.device("cuda", device_index)
        handle = C.c_void_p()
        rc = self.lib.pdb_create(C.byref(handle), device_index)
        if rc != 0:
            raise NativeError(f"pdb_create({device_index}) failed: {self.lib.pdb_last_error(None).decode()}")
        self.handle = handle
        self.weights_key = None
        self.ggs_layout = {v: k for k, v in GGS_LAYOUTS.items()}[int(self.lib.pdb_ggs_layout_get(handle))]

    @classmethod
    def get(cls, device) -> "Context":
        if not torch.cuda.is_available():
            raise NativeError("no CUDA device: posediffusion_b200 runs on H100 (sm_90a) only, there is no CPU fallback")
        device = torch.device(device)
        index = device.index if device.index is not None else torch.cuda.current_device()
        if index not in cls._by_device:
            cls._by_device[index] = Context(index)
        return cls._by_device[index]

    def _ok(self, rc: int, what: str):
        if rc != 0:
            raise NativeError(f"{what} failed ({rc}): {self.lib.pdb_last_error(self.handle).decode()}")

    @property
    def launch_count(self) -> int:
        return int(self.lib.pdb_launch_count(self.handle))

    def profile(self, on: bool):
        self._ok(self.lib.pdb_profile_enable(self.handle, int(on)), "pdb_profile_enable")

    def profile_read(self):
        """(ggs_ms, ggs_launches, denoiser_ms, denoiser_launches) since the last read; synchronises."""
        a, b, c, d = C.c_double(), C.c_int64(), C.c_double(), C.c_int64()
        self._ok(self.lib.pdb_profile_read(self.handle, C.byref(a), C.byref(b), C.byref(c), C.byref(d)), "pdb_profile_read")
        return a.value, b.value, c.value, d.value

    def ggs_clocks(self, enable=True, read: bool = False):
        """Stage timing probe: enable = True / 1 for the GGS kernel, 2 for the fp32 denoiser kernel (same buffer)."""
        out = np.zeros((256, 8), dtype=np.int64) if read else None
        self._ok(self.lib.pdb_debug_ggs_clocks(self.handle, int(enable), out.ctypes.data if read else None, 256), "pdb_debug_ggs_clocks")
        return out

    def set_denoiser_engine(self, mode: str = "auto"):
        """'auto' (fp32 kernel below 128 tokens, tensor cores above), 'fp32' or 'tf32'."""
        self._ok(self.lib.pdb_denoiser_engine(self.handle, {"auto": 0, "fp32": 1, "tf32": 2}[mode]), "pdb_denoiser_engine")

    def set_denoiser_handover(self, flagged: bool):
        """Stage hand-over of the persistent fp32 denoiser kernel: group barriers (default) or flag-carrying words."""
        self._ok(self.lib.pdb_debug_denoiser_handover(self.handle, int(flagged)), "pdb_debug_denoiser_handover")

    def set_tc_swap(self, on: bool):
        """Swap-AB tensor-core tiles for GEMMs with at most 96 tokens (default off)."""
        self._ok(self.lib.pdb_debug_tc_swap(self.handle, int(on)), "pdb_debug_tc_swap")

    def set_ggs_layout(self, layout: str = "plain"):
        """Stream layout of match sets packed from now on: 'plain' (default) or 'paired' (csrc/ggs_layout.cuh; experimental)."""
        self._ok(self.lib.pdb_ggs_layout(self.handle, GGS_LAYOUTS[layout]), "pdb_ggs_layout")
        self.ggs_layout = layout

    def tc_linear(self, x: torch.Tensor, w: torch.Tensor, bias=None, residual=None, relu: bool = False,
                  in_place: bool = False) -> torch.Tensor:
        """Y = relu?(x @ w^T + bias + residual) on the tensor cores (wgmma, TF32 products, fp32 accumulate).
        in_place: Y is the residual buffer itself (the denoiser's residual-stream update; small problems then split K)."""
        S, K = x.shape
        O = w.shape[0]
        if in_place and residual is None:
            raise ValueError("in_place needs a residual")
        y = residual if in_place else torch.empty(S, O, device=self.device)
        self._ok(self.lib.pdb_debug_tc_linear(self.handle, x.data_ptr(), w.data_ptr(), bias.data_ptr() if bias is not None else None,
                                              residual.data_ptr() if residual is not None else None, y.data_ptr(), S, O, K,
                                              int(relu), _stream_ptr(self.device)), "pdb_debug_tc_linear")
        return y

    def sm_count(self) -> int:
        sm, a, b = C.c_int32(), C.c_int32(), C.c_int32()
        self.lib.pdb_device_info(self.handle, C.byref(sm), C.byref(a), C.byref(b))
        return sm.value

    # ---- weights --------------------------------------------------------------------------------
    def load_denoiser(self, tensors: Sequence[torch.Tensor]):
        if len(tensors) != PDB_NUM_WEIGHT_TENSORS:
            raise NativeError(f"expected {PDB_NUM_WEIGHT_TENSORS} tensors, got {len(tensors)}")
        keep = [t.detach().to(dtype=torch.float32).contiguous() for t in tensors]
        arr = (C.c_void_p * len(keep))(*[C.c_void_p(t.data_ptr()) for t in keep])
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_denoiser_load(self.handle, arr, len(keep), _stream_ptr(self.device)), "pdb_denoiser_load")

    # ---- training ------------------------------------------------------------------------------------
    def _tensor_array(self, tensors: Sequence[torch.Tensor], count: int, what: str):
        if len(tensors) != count:
            raise NativeError(f"expected {count} tensors, got {len(tensors)}")
        for i, p in enumerate(tensors):
            _check_dev(p, f"{what} {i}", self.device)
        return (C.c_void_p * len(tensors))(*[C.c_void_p(p.data_ptr()) for p in tensors])

    def train_forward(self, params: Sequence[torch.Tensor], x_start, t, noise, z, dropout_p: float, seed: int, loss_type: str):
        """p_losses forward: returns (workspace, loss, x_t, x0).  The workspace holds what train_backward needs; it belongs to
        the caller (one per outstanding forward)."""
        B, N, _ = x_start.shape
        for name, v, shape in (("x_start", x_start, (B, N, TARGET_DIM)), ("noise", noise, (B, N, TARGET_DIM)), ("z", z, (B, N, Z_DIM))):
            _check_dev(v, name, self.device, shape)
        if t.dtype != torch.int32 or tuple(t.shape) != (B,) or t.device != self.device or not t.is_contiguous():
            raise NativeError(f"t must be a contiguous int32 [{B}] tensor on {self.device}")
        if N > TRAIN_MAX_FRAMES:
            raise NativeError(f"training supports at most {TRAIN_MAX_FRAMES} frames per sequence, got {N}")
        nbytes = train_workspace_bytes(B, N)
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=self.device)
        loss, x_t, x0 = torch.empty_like(x_start), torch.empty_like(x_start), torch.empty_like(x_start)
        arr = self._tensor_array(params, PDB_NUM_WEIGHT_TENSORS, "parameter")
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_train_forward(self.handle, arr, x_start.data_ptr(), t.data_ptr(), noise.data_ptr(), z.data_ptr(), B, N,
                                                float(dropout_p), int(seed) & (2**64 - 1), LOSS_TYPES[loss_type], ws.data_ptr(),
                                                loss.data_ptr(), x_t.data_ptr(), x0.data_ptr(), _stream_ptr(self.device)),
                     "pdb_train_forward")
        return ws, loss, x_t, x0

    def train_backward(self, params: Sequence[torch.Tensor], ws: torch.Tensor, grad_loss: Optional[torch.Tensor],
                       grad_x0: Optional[torch.Tensor], grad_z: Optional[torch.Tensor] = None) -> List[torch.Tensor]:
        """Gradients of the 108 parameters; with `grad_z` (a [B,N,384] buffer) also dL/dz, written into it."""
        arr = self._tensor_array(params, PDB_NUM_WEIGHT_TENSORS, "parameter")
        grads = [torch.empty_like(p) for p in params]
        garr = (C.c_void_p * len(grads))(*[C.c_void_p(g.data_ptr()) for g in grads])
        gl = grad_loss.data_ptr() if grad_loss is not None else None
        gx = grad_x0.data_ptr() if grad_x0 is not None else None
        with torch.cuda.device(self.device):
            if grad_z is None:
                self._ok(self.lib.pdb_train_backward(self.handle, arr, ws.data_ptr(), gl, gx, garr, _stream_ptr(self.device)),
                         "pdb_train_backward")
            else:
                _check_dev(grad_z, "grad_z", self.device)
                self._ok(self.lib.pdb_train_backward_z(self.handle, arr, ws.data_ptr(), gl, gx, garr, grad_z.data_ptr(),
                                                       _stream_ptr(self.device)), "pdb_train_backward_z")
        return grads

    def camera_to_pose(self, R: torch.Tensor, T: torch.Tensor, focal: torch.Tensor, log_focal_length_bias=1.8, min_focal_length=0.1,
                       max_focal_length=20.0) -> torch.Tensor:
        """R [..., 3, 3], T [..., 3], focal [..., 2] -> pose [..., 9] (absT_quaR_logFL)."""
        lead = tuple(T.shape[:-1])
        Rf = R.reshape(-1, 3, 3).to(torch.float32).contiguous()
        Tf = T.reshape(-1, 3).to(torch.float32).contiguous()
        Ff = focal.reshape(-1, 2).to(torch.float32).contiguous()
        n = Tf.shape[0]
        for v, name, shape in ((Rf, "R", (n, 3, 3)), (Tf, "T", (n, 3)), (Ff, "focal_length", (n, 2))):
            _check_dev(v, name, self.device, shape)
        pose = torch.empty((n, TARGET_DIM), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_camera_to_pose(self.handle, Rf.data_ptr(), Tf.data_ptr(), Ff.data_ptr(), n, float(log_focal_length_bias),
                                                 float(min_focal_length), float(max_focal_length), pose.data_ptr(),
                                                 _stream_ptr(self.device)), "pdb_camera_to_pose")
        return pose.reshape(*lead, TARGET_DIM)

    # ---- post-loop geometry ---------------------------------------------------------------------------
    def pose_to_camera(self, pose: torch.Tensor, log_focal_length_bias=1.8, min_focal_length=0.1, max_focal_length=20.0):
        """pose [..., 9] -> (R [n,3,3], T [n,3], focal [n,2]) with n = prod(leading dims)."""
        flat = pose.reshape(-1, TARGET_DIM).to(torch.float32).contiguous()
        _check_dev(flat, "pose", self.device)
        n = flat.shape[0]
        R = torch.empty((n, 3, 3), device=self.device, dtype=torch.float32)
        T = torch.empty((n, 3), device=self.device, dtype=torch.float32)
        F = torch.empty((n, 2), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_pose_to_camera(self.handle, C.c_void_p(flat.data_ptr()), n, float(log_focal_length_bias),
                                                 float(min_focal_length), float(max_focal_length), C.c_void_p(R.data_ptr()),
                                                 C.c_void_p(T.data_ptr()), C.c_void_p(F.data_ptr()), _stream_ptr(self.device)), "pdb_pose_to_camera")
        return R, T, F

    def rel_pose_error(self, R_pred, T_pred, R_gt, T_gt, batch: int):
        """(r_deg, t_deg) [batch * N(N-1)/2] for `batch` sequences of N cameras; raises ValueError like pytorch3d's
        so3_rotation_angle when a relative rotation has a trace outside the valid range."""
        tensors = [t.to(torch.float32).contiguous() for t in (R_pred, T_pred, R_gt, T_gt)]
        total = tensors[0].shape[0]
        if batch < 1 or total % batch:
            raise NativeError(f"{total} cameras do not split into {batch} sequences")
        frames = total // batch
        for t, name, shape in zip(tensors, ("R_pred", "T_pred", "R_gt", "T_gt"), ((total, 3, 3), (total, 3), (total, 3, 3), (total, 3))):
            _check_dev(t, name, self.device, shape)
        pairs = batch * frames * (frames - 1) // 2
        r = torch.empty(pairs, device=self.device, dtype=torch.float32)
        t = torch.empty(pairs, device=self.device, dtype=torch.float32)
        flag = torch.zeros(1, device=self.device, dtype=torch.int32)
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_rel_pose_error(self.handle, *[C.c_void_p(x.data_ptr()) for x in tensors], batch, frames,
                                                 C.c_void_p(r.data_ptr()), C.c_void_p(t.data_ptr()), C.c_void_p(flag.data_ptr()),
                                                 _stream_ptr(self.device)), "pdb_rel_pose_error")
        if int(flag.item()):
            raise ValueError("A matrix has trace outside valid range [-1-eps,3+eps].")
        return r, t

    def cameras_align(self, R_src, T_src, R_tgt, T_tgt, estimate_scale: bool = True, eps: float = 1e-9):
        """corresponding_cameras_alignment(mode="extrinsics") -> (R_aligned [n,3,3], T_aligned [n,3], align [13] = R | T | scale)."""
        tensors = [t.to(torch.float32).contiguous() for t in (R_src, T_src, R_tgt, T_tgt)]
        n = tensors[0].shape[0]
        for t, name, shape in zip(tensors, ("R_src", "T_src", "R_tgt", "T_tgt"), ((n, 3, 3), (n, 3), (n, 3, 3), (n, 3))):
            _check_dev(t, name, self.device, shape)
        R = torch.empty((n, 3, 3), device=self.device, dtype=torch.float32)
        T = torch.empty((n, 3), device=self.device, dtype=torch.float32)
        align = torch.empty(13, device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_cameras_align(self.handle, *[C.c_void_p(x.data_ptr()) for x in tensors], n, int(bool(estimate_scale)),
                                                float(eps), C.c_void_p(R.data_ptr()), C.c_void_p(T.data_ptr()),
                                                C.c_void_p(align.data_ptr()), _stream_ptr(self.device)), "pdb_cameras_align")
        return R, T, align

    def load_vit(self, tensors: Sequence[torch.Tensor]):
        """DINO ViT-S/16 parameters in hub state_dict order (150 tensors, host or this device)."""
        if len(tensors) != PDB_VIT_NUM_TENSORS:
            raise NativeError(f"expected {PDB_VIT_NUM_TENSORS} tensors, got {len(tensors)}")
        on_device = all(t.is_cuda for t in tensors)
        keep = [t.detach().to(dtype=torch.float32).contiguous() if on_device else t.detach().to("cpu", torch.float32).contiguous()
                for t in tensors]
        arr = (C.c_void_p * len(keep))(*[C.c_void_p(t.data_ptr()) for t in keep])
        numels = (C.c_int64 * len(keep))(*[t.numel() for t in keep])
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_vit_load(self.handle, arr, numels, len(keep), int(on_device), _stream_ptr(self.device)), "pdb_vit_load")
        self.vit_key = None

    def extract_features(self, images: torch.Tensor, scale_factors: Sequence[float], debug_stage: Optional[int] = None):
        """images [n,3,H,W] in [0,1] -> z [n,384]; with debug_stage also the residual stream after that stage."""
        n, ch, H, W = images.shape
        if ch != 3:
            raise NativeError(f"images must be [n,3,H,W], got {tuple(images.shape)}")
        _check_dev(images, "images", self.device)
        sf = (C.c_double * len(scale_factors))(*[float(f) for f in scale_factors])
        z = torch.empty((n, VIT_DIM), device=self.device, dtype=torch.float32)
        dbg = None
        if debug_stage is not None:
            rows = 0
            for f in scale_factors:
                oh, ow = (H, W) if f == 1 else (int(np.floor(H * float(f))), int(np.floor(W * float(f))))
                rows += n * (1 + (oh // 16) * (ow // 16))
            dbg = torch.empty((rows, VIT_DIM), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_extract_features(self.handle, C.c_void_p(images.data_ptr()), n, H, W, sf, len(scale_factors),
                                                   C.c_void_p(z.data_ptr()), C.c_void_p(dbg.data_ptr()) if dbg is not None else None,
                                                   int(debug_stage or 0), _stream_ptr(self.device)), "pdb_extract_features")
        return (z, dbg) if debug_stage is not None else z

    # ---- backbone training ----------------------------------------------------------------------------
    def vit_train_workspace_bytes(self, n_images: int, height: int, width: int, scale_factors: Sequence[float]) -> int:
        return vit_train_workspace_bytes(n_images, height, width, scale_factors)

    def vit_train_forward(self, params: Sequence[torch.Tensor], images: torch.Tensor, scale_factors: Sequence[float]):
        """Backbone forward that keeps what vit_backward needs: returns (workspace, z [n,384]).  The workspace belongs to the
        caller (one per outstanding forward).  `params`: the 150 tensors in hub state_dict order, on this device."""
        n, ch, H, W = images.shape
        if ch != 3:
            raise NativeError(f"images must be [n,3,H,W], got {tuple(images.shape)}")
        _check_dev(images, "images", self.device)
        nbytes = vit_train_workspace_bytes(n, H, W, scale_factors)
        if nbytes <= 0:
            raise NativeError(f"unsupported backbone training shape: {n} images of {H}x{W} at scales {list(scale_factors)}")
        arr = self._tensor_array(params, PDB_VIT_NUM_TENSORS, "parameter")
        sf = (C.c_double * len(scale_factors))(*[float(f) for f in scale_factors])
        ws = torch.empty(nbytes // 4, dtype=torch.float32, device=self.device)
        z = torch.empty((n, VIT_DIM), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_vit_train_forward(self.handle, arr, images.data_ptr(), n, H, W, sf, len(scale_factors), ws.data_ptr(),
                                                    z.data_ptr(), _stream_ptr(self.device)), "pdb_vit_train_forward")
        return ws, z

    def vit_backward(self, params: Sequence[torch.Tensor], ws: torch.Tensor, grad_z: torch.Tensor) -> List[torch.Tensor]:
        """d(sum(grad_z * z)) / d params for the forward held in `ws`."""
        arr = self._tensor_array(params, PDB_VIT_NUM_TENSORS, "parameter")
        _check_dev(grad_z, "grad_z", self.device)
        grads = [torch.empty_like(p) for p in params]
        garr = (C.c_void_p * len(grads))(*[C.c_void_p(g.data_ptr()) for g in grads])
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_vit_backward(self.handle, arr, ws.data_ptr(), grad_z.data_ptr(), garr, _stream_ptr(self.device)),
                     "pdb_vit_backward")
        return grads

    def extract_features_host(self, images: np.ndarray, scale_factors: Sequence[float]) -> np.ndarray:
        n, ch, H, W = images.shape
        if ch != 3 or images.dtype != np.float32 or not images.flags.c_contiguous:
            raise NativeError("images must be contiguous float32 [n,3,H,W]")
        sf = (C.c_double * len(scale_factors))(*[float(f) for f in scale_factors])
        z = np.empty((n, VIT_DIM), dtype=np.float32)
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_extract_features_host(self.handle, images.ctypes.data_as(C.c_void_p), n, H, W, sf, len(scale_factors),
                                                        z.ctypes.data_as(C.c_void_p), _stream_ptr(self.device)), "pdb_extract_features_host")
        return z

    def preprocess_images(self, frames: Sequence[np.ndarray], crops: Sequence[Sequence[int]], out_size: int) -> torch.Tensor:
        """Decoded frames (uint8 [H,W,3] each, sizes may differ) and their square crops {top, left, side} -> float32
        [n,3,out_size,out_size] on this device: crop / 255 resized bilinearly (pdb_images_preprocess_host)."""
        keep = [np.ascontiguousarray(f, dtype=np.uint8) for f in frames]
        for i, f in enumerate(keep):
            if f.ndim != 3 or f.shape[2] != 3:
                raise NativeError(f"frame {i} has shape {f.shape}, expected [H, W, 3] uint8")
        n = len(keep)
        ptrs = (C.c_void_p * max(n, 1))(*[f.ctypes.data for f in keep])
        hw = np.asarray([f.shape[:2] for f in keep] or np.zeros((0, 2)), dtype=np.int32).reshape(-1, 2)
        crop = np.ascontiguousarray(np.asarray(crops, dtype=np.int32).reshape(-1, 3))
        if len(crop) != n:
            raise NativeError(f"{len(crop)} crops for {n} frames")
        images = torch.empty((n, 3, max(int(out_size), 0), max(int(out_size), 0)), device=self.device, dtype=torch.float32)
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_images_preprocess_host(self.handle, n, ptrs, hw.ctypes.data, crop.ctypes.data, int(out_size),
                                                         C.c_void_p(images.data_ptr()), _stream_ptr(self.device)),
                     "pdb_images_preprocess_host")
        return images

    # ---- denoiser / sampler -----------------------------------------------------------------------
    def denoiser_forward(self, x: torch.Tensor, t: int, z: torch.Tensor) -> torch.Tensor:
        B, N, _ = x.shape
        _check_dev(x, "x", self.device, (B, N, TARGET_DIM))
        _check_dev(z, "z", self.device, (B, N, Z_DIM))
        eps = torch.empty_like(x)
        self._ok(self.lib.pdb_denoiser_forward(self.handle, x.data_ptr(), int(t), z.data_ptr(), B, N, eps.data_ptr(),
                                               _stream_ptr(self.device)), "pdb_denoiser_forward")
        return eps

    def p_sample(self, x, t: int, z, noise: Optional[torch.Tensor]):
        B, N, _ = x.shape
        _check_dev(x, "x", self.device, (B, N, TARGET_DIM))
        _check_dev(z, "z", self.device, (B, N, Z_DIM))
        if noise is not None:
            _check_dev(noise, "noise", self.device, (B, N, TARGET_DIM))
        pred, mean, x0 = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
        self._ok(self.lib.pdb_p_sample(self.handle, x.data_ptr(), int(t), z.data_ptr(),
                                       noise.data_ptr() if noise is not None else None, B, N, pred.data_ptr(),
                                       mean.data_ptr(), x0.data_ptr(), _stream_ptr(self.device)), "pdb_p_sample")
        return pred, mean, x0

    # ---- correspondences ------------------------------------------------------------------------
    def pack_matches(self, matches_dict: Dict) -> Matches:
        frames, _, height, width = (int(v) for v in matches_dict["img_shape"])
        kp1 = np.ascontiguousarray(matches_dict["kp1"], dtype=np.float64).reshape(-1, 2)
        kp2 = np.ascontiguousarray(matches_dict["kp2"], dtype=np.float64).reshape(-1, 2)
        i12 = np.ascontiguousarray(matches_dict["i12"], dtype=np.int64).reshape(-1, 2)
        if not (len(kp1) == len(kp2) == len(i12)):
            raise ValueError("kp1, kp2 and i12 must have the same number of rows")
        handle = C.c_void_p()
        with torch.cuda.device(self.device):
            rc = self.lib.pdb_matches_pack(self.handle, kp1.ctypes.data, kp2.ctypes.data, i12.ctypes.data, len(kp1),
                                           frames, height, width, 0, _stream_ptr(self.device), C.byref(handle))
        if rc == -1:
            raise ValueError(self.lib.pdb_last_error(self.handle).decode())
        self._ok(rc, "pdb_matches_pack")
        return Matches(self, handle, frames, len(kp1))

    def sampson_eval(self, matches: Matches, pose: torch.Tensor, update_R=True, update_T=True, update_FL=True,
                     sampson_max: float = 10.0, dump: bool = False):
        _check_dev(pose, "pose", self.device, (matches.frames, TARGET_DIM))
        grad = torch.empty_like(pose)
        scalars = torch.zeros(4, device=self.device)
        Fd = torch.zeros(max(matches.segments, 1), 9, device=self.device) if dump else None
        Gd = torch.zeros(max(matches.segments, 1), 9, device=self.device) if dump else None
        self._ok(self.lib.pdb_sampson_eval(self.handle, matches.handle, pose.data_ptr(), int(update_R), int(update_T),
                                           int(update_FL), float(sampson_max), grad.data_ptr(), scalars.data_ptr(),
                                           Fd.data_ptr() if dump else None, Gd.data_ptr() if dump else None,
                                           _stream_ptr(self.device)), "pdb_sampson_eval")
        return grad, scalars, Fd, Gd

    def _problem_array(self, problems: Sequence[Matches]):
        return (C.c_void_p * len(problems))(*[p.handle for p in problems])

    @staticmethod
    def _check_problems(problems: Sequence[Matches], batch: int, frames: int):
        """One match set per sequence, each packed for the pose's frame count (the library checks the same)."""
        if len(problems) != batch:
            raise ValueError(f"{len(problems)} match sets for a batch of {batch} sequences")
        for i, p in enumerate(problems):
            if p.frames != frames:
                raise ValueError(f"match set {i} has img_shape[0] = {p.frames}, the sequence has {frames} frames")

    def ggs(self, problems: Sequence[Matches], pose: torch.Tensor, cfg: Dict, want_stats: bool = True):
        """In-place geometry-guided sampling on pose [B, N, 9]; returns a device stats tensor (uint8 view) or None."""
        B = len(problems)
        _check_dev(pose, "model_mean", self.device, (B, problems[0].frames, TARGET_DIM))
        stats = torch.zeros(B * GGS_STATS_DTYPE.itemsize, dtype=torch.uint8, device=self.device) if want_stats else None
        conf = ggs_config_struct(cfg)
        self._ok(self.lib.pdb_ggs(self.handle, self._problem_array(problems), B, pose.data_ptr(), C.byref(conf),
                                  stats.data_ptr() if want_stats else None, _stream_ptr(self.device)), "pdb_ggs")
        return stats

    def _device_loop(self, entry: str, ddim_args, z: torch.Tensor, draws: torch.Tensor, draw_slots: int, trail_slots: int,
                     stats_rows: int, problems, cfg, cond_start_step: int, want_trail: bool, want_stats: bool):
        """Check the shapes, allocate pose [B, N, 9], trail [trail_slots, B, N, 9] and stats [stats_rows, B] and run the device
        entry `entry` (`ddim_args` go between the frame count and the match sets)."""
        B, N, _ = z.shape
        _check_dev(z, "z", self.device, (B, N, Z_DIM))
        _check_dev(draws, "draws", self.device, (draw_slots, B, N, TARGET_DIM))
        if problems:
            self._check_problems(problems, B, N)
        pose = torch.empty(B, N, TARGET_DIM, device=self.device)
        trail = torch.empty(trail_slots, B, N, TARGET_DIM, device=self.device) if want_trail else None
        stats = None
        if want_stats and problems and stats_rows:
            stats = torch.zeros(stats_rows * B * GGS_STATS_DTYPE.itemsize, dtype=torch.uint8, device=self.device)
        conf = ggs_config_struct(cfg) if problems else None
        self._ok(getattr(self.lib, entry)(self.handle, z.data_ptr(), draws.data_ptr(), B, N, *ddim_args,
                                          self._problem_array(problems) if problems else None, len(problems) if problems else 0,
                                          C.byref(conf) if conf is not None else None, int(cond_start_step), pose.data_ptr(),
                                          trail.data_ptr() if want_trail else None, stats.data_ptr() if stats is not None else None,
                                          _stream_ptr(self.device)), entry)
        return pose, trail, stats

    def sample_loop(self, z: torch.Tensor, draws: torch.Tensor, problems: Optional[Sequence[Matches]], cfg: Optional[Dict],
                    cond_start_step: int, want_trail: bool = True, want_stats: bool = True):
        guided = clamp_guided(cond_start_step) if problems else 0
        return self._device_loop("pdb_sample_loop", (), z, draws, NUM_TIMESTEPS + 1, NUM_TIMESTEPS + 1, guided, problems, cfg,
                                 cond_start_step, want_trail, want_stats)

    def sample_loop_ddim(self, z: torch.Tensor, draws: torch.Tensor, steps: int, eta: float, problems: Optional[Sequence[Matches]],
                         cfg: Optional[Dict], cond_start_step: int, want_trail: bool = True, want_stats: bool = True,
                         guided_steps: Optional[int] = None):
        """pdb_sample_loop_ddim_guided: (pose, trail [1 + steps, B, N, 9] or None, stats [g', B] records).  The guided tail over
        g = clamp(cond_start_step) timesteps takes g' = `guided_steps` (default g) jumps, the prefix k = steps - g'.  draws
        [1 + k, B, N, 9] for eta > 0, [1, B, N, 9] for eta == 0.  Without problems and with cond_start_step > 0 only the prefix runs
        (pose = x_{g-1})."""
        guided = clamp_guided(cond_start_step)
        k = ddim_check(steps, guided, eta, guided_steps)
        gs = guided if guided_steps is None else int(guided_steps)
        return self._device_loop("pdb_sample_loop_ddim_guided", (int(steps), float(eta), gs), z, draws, 1 + k if eta > 0 else 1,
                                 1 + int(steps), gs, problems, cfg, cond_start_step, want_trail, want_stats)

    @staticmethod
    def _check_host_buffers(z: np.ndarray, draws: np.ndarray, draw_slots: int, trail_out, trail_slots: int, stats_out, stats_rows: int):
        """The host arrays of a host-buffer entry against the loop's slot counts (the library trusts their sizes)."""
        B, N, _ = z.shape
        want = (draw_slots, B, N, TARGET_DIM)
        if draws.shape != want or draws.dtype != np.float32 or not draws.flags.c_contiguous:
            raise ValueError(f"draws must be C-contiguous float32 {want}, got {draws.shape}")
        if trail_out is not None and trail_out.shape != (trail_slots, B, N, TARGET_DIM):
            raise ValueError(f"trail_out must be {(trail_slots, B, N, TARGET_DIM)}, got {trail_out.shape}")
        if stats_out is not None and stats_out.nbytes < stats_rows * B * GGS_STATS_DTYPE.itemsize:
            raise ValueError(f"stats_out needs {stats_rows * B} records")

    def sample_loop_host(self, z: np.ndarray, draws: np.ndarray, problems, cfg, cond_start_step: int,
                         pose_out: np.ndarray, trail_out: Optional[np.ndarray] = None, stats_out: Optional[np.ndarray] = None):
        """Host-buffer entry (numpy float32 arrays, ideally pinned): the end-to-end call bench.py times."""
        B, N, _ = z.shape
        guided = clamp_guided(cond_start_step) if problems else 0
        self._check_host_buffers(z, draws, NUM_TIMESTEPS + 1, trail_out, NUM_TIMESTEPS + 1, stats_out, guided)
        if problems:
            self._check_problems(problems, B, N)
        conf = ggs_config_struct(cfg) if problems else None
        with torch.cuda.device(self.device):
            self._ok(self.lib.pdb_sample_loop_host(self.handle, z.ctypes.data, draws.ctypes.data, B, N,
                                                   self._problem_array(problems) if problems else None,
                                                   len(problems) if problems else 0,
                                                   C.byref(conf) if conf is not None else None, int(cond_start_step),
                                                   pose_out.ctypes.data, trail_out.ctypes.data if trail_out is not None else None,
                                                   stats_out.ctypes.data if stats_out is not None else None,
                                                   _stream_ptr(self.device)), "pdb_sample_loop_host")
        return pose_out

    def _host_matches_loop(self, entry: str, ddim_args, z: np.ndarray, draws: np.ndarray, draw_slots: int, trail_slots: int,
                           stats_rows: int, matches_dicts, cfg, cond_start_step: int, pose_out, trail_out, stats_out):
        B, N, _ = z.shape
        self._check_host_buffers(z, draws, draw_slots, trail_out, trail_slots, stats_out, stats_rows)
        ptrs, counts, shape, _keep = self._host_match_arrays(matches_dicts, B, N)
        conf = ggs_config_struct(cfg)
        with torch.cuda.device(self.device):
            rc = getattr(self.lib, entry)(self.handle, z.ctypes.data, draws.ctypes.data, B, N, *ddim_args, ptrs[0], ptrs[1], ptrs[2],
                                          counts, shape[0], shape[1], C.byref(conf), int(cond_start_step), pose_out.ctypes.data,
                                          trail_out.ctypes.data if trail_out is not None else None,
                                          stats_out.ctypes.data if stats_out is not None else None, _stream_ptr(self.device))
        if rc == -1:
            raise ValueError(self.lib.pdb_last_error(self.handle).decode())
        self._ok(rc, entry)
        return pose_out

    def sample_loop_host_matches(self, z: np.ndarray, draws: np.ndarray, matches_dicts, cfg, cond_start_step: int,
                                 pose_out: np.ndarray, trail_out: Optional[np.ndarray] = None, stats_out: Optional[np.ndarray] = None):
        """The end-to-end call from the reference's matches_dict format (one dict per sequence): the match sets are packed and
        uploaded while the unguided steps already run (pdb_sample_loop_host_matches)."""
        return self._host_matches_loop("pdb_sample_loop_host_matches", (), z, draws, NUM_TIMESTEPS + 1, NUM_TIMESTEPS + 1,
                                       clamp_guided(cond_start_step), matches_dicts, cfg, cond_start_step, pose_out, trail_out,
                                       stats_out)

    def sample_loop_host_matches_ddim(self, z: np.ndarray, draws: np.ndarray, matches_dicts, cfg, cond_start_step: int, steps: int,
                                      eta: float, pose_out: np.ndarray, trail_out: Optional[np.ndarray] = None,
                                      stats_out: Optional[np.ndarray] = None, guided_steps: Optional[int] = None):
        """sample_loop_host_matches on the DDIM loop of sample_loop_ddim (pdb_sample_loop_host_matches_ddim): draws [1 + k, B, N, 9]
        for eta > 0, [1, B, N, 9] for eta == 0; trail_out [1 + steps, B, N, 9]; stats_out g' records per sequence."""
        guided = clamp_guided(cond_start_step)
        k = ddim_check(steps, guided, eta, guided_steps)
        gs = guided if guided_steps is None else int(guided_steps)
        return self._host_matches_loop("pdb_sample_loop_host_matches_ddim", (int(steps), float(eta), gs), z, draws,
                                       1 + k if eta > 0 else 1, 1 + int(steps), gs, matches_dicts, cfg, cond_start_step, pose_out,
                                       trail_out, stats_out)

    @staticmethod
    def _host_match_arrays(matches_dicts, B: int, N: int):
        """The pointer arrays of pdb_sample_loop_host_matches* for one matches_dict per sequence, and the arrays they point into."""
        if len(matches_dicts) != B:
            raise ValueError(f"{len(matches_dicts)} match sets for a batch of {B} sequences (one per sequence)")
        keep, shape = [], None
        for md in matches_dicts:
            frames, _, height, width = (int(v) for v in md["img_shape"])
            if frames != N:
                raise ValueError(f"match set of {frames} frames used with {N} frames")
            if shape is not None and shape != (height, width):
                raise ValueError("all sequences of one call must share the image size")
            shape = (height, width)
            kp1 = np.ascontiguousarray(md["kp1"], dtype=np.float64).reshape(-1, 2)
            kp2 = np.ascontiguousarray(md["kp2"], dtype=np.float64).reshape(-1, 2)
            i12 = np.ascontiguousarray(md["i12"], dtype=np.int64).reshape(-1, 2)
            if not (len(kp1) == len(kp2) == len(i12)):
                raise ValueError("kp1, kp2 and i12 must have the same number of rows")
            keep.append((kp1, kp2, i12))
        ptrs = [(C.c_void_p * B)(*[k[j].ctypes.data for k in keep]) for j in range(3)]
        counts = (C.c_int64 * B)(*[len(k[0]) for k in keep])
        return ptrs, counts, shape, keep


def stats_to_numpy(stats: Optional[torch.Tensor]) -> Optional[np.ndarray]:
    """Device stats bytes -> structured numpy array (synchronises)."""
    if stats is None:
        return None
    return stats.cpu().numpy().view(GGS_STATS_DTYPE)
