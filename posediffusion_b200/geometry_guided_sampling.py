"""`geometry_guided_sampling` with the reference's signature (util/geometry_guided_sampling.py:14),
running all five GGS_optimize phases in one persistent sm_90a kernel launch.

    cond_fn = partial(geometry_guided_sampling, matches_dict=matches_dict, GGS_cfg=GGS_cfg)   # demo.py:89
    model_mean = cond_fn(model_mean, t)

`matches_dict` is the reference's dict (kp1/kp2 float64 [M,2], i12 int64 [M,2], img_shape); for a batch of
B > 1 sequences pass a list of B such dicts (the reference's own GGS is only meaningful for B = 1,
SURVEY.md §0 row 5).  Matches are packed and uploaded ONCE per dict (the reference re-uploads 48 B/match
on every guided step, :19-24) and cached per dict object, keyed on the identity of its arrays plus a sampled content
fingerprint; `invalidate_matches(d)` drops the device copy after an in-place edit.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, List, Sequence, Union

import numpy as np
import torch

from . import _native

_KEEP: "OrderedDict[int, tuple]" = OrderedDict()
_KEEP_MAX = 8  # packed sets pinned on the GPU at most (least recently used goes first)


def _fingerprint(a) -> tuple:
    """Cheap content tag of a match array: shape, dtype and 64 strided samples (a full checksum of a 778 240-row set costs
    more than packing it).  Catches a different set behind a recycled object id and most in-place edits; call
    `invalidate_matches` after editing `kp1` / `kp2` / `i12` in place to be certain."""
    a = np.asarray(a)
    flat = a.reshape(-1)
    step = max(1, flat.size // 64)
    return (a.shape, a.dtype.str, flat[::step][:64].tobytes(), flat[-1:].tobytes())


def invalidate_matches(matches_dict: Union[Dict, Sequence[Dict], None] = None) -> None:
    """Forget the device copy of `matches_dict` (all cached sets if None): the next call packs and uploads it again, as the
    reference does on every call (util/geometry_guided_sampling.py:19-24)."""
    if matches_dict is None:
        _KEEP.clear()
        return
    for d in ([matches_dict] if isinstance(matches_dict, dict) else list(matches_dict)):
        _KEEP.pop(id(d), None)


def packed_matches(ctx: "_native.Context", matches_dict: Union[Dict, Sequence[Dict]]) -> List["_native.Matches"]:
    dicts = [matches_dict] if isinstance(matches_dict, dict) else list(matches_dict)
    out = []
    for d in dicts:
        arrays = (d["kp1"], d["kp2"], d["i12"])
        key = (ctx.device.index, ctx.ggs_layout, tuple(id(a) for a in arrays), tuple(d["img_shape"]),
               tuple(_fingerprint(a) for a in arrays))
        hit = _KEEP.get(id(d))
        if hit is None or hit[0] != key:
            # the entry holds the source arrays: their ids cannot be recycled for other data while it is cached
            hit = (key, ctx.pack_matches(d), arrays)
            _KEEP[id(d)] = hit
            while len(_KEEP) > _KEEP_MAX:
                _KEEP.popitem(last=False)
        _KEEP.move_to_end(id(d))
        out.append(hit[1])
    return out


def format_log(t: int, stats_row) -> List[str]:
    """The reference's prints (:107, :124), reconstructed from the device-side statistics."""
    lines = []
    for phase in range(_native.PDB_GGS_PHASES):
        if stats_row["dropped"][phase]:
            lines.append("Drop this pair because of insufficient valid matches")
        lines.append(f"t={t:02d} | sampson={float(stats_row['sampson'][phase]):05f}")
    return lines


def geometry_guided_sampling(model_mean: torch.Tensor, t: int, matches_dict, GGS_cfg: Dict):
    if model_mean.dim() != 3 or model_mean.shape[-1] != _native.TARGET_DIM:
        raise ValueError("model_mean must be [B, N, 9]")
    ctx = _native.Context.get(model_mean.device)
    problems = packed_matches(ctx, matches_dict)
    if len(problems) != model_mean.shape[0]:
        raise ValueError(f"{len(problems)} match sets for a batch of {model_mean.shape[0]} sequences")
    pose = model_mean.detach()
    if pose.dtype != torch.float32 or not pose.is_contiguous():
        pose = pose.float().contiguous()
    verbose = bool(GGS_cfg.get("verbose", True))
    stats = ctx.ggs(problems, pose, GGS_cfg, want_stats=verbose)
    if verbose:  # one device->host read per call (the reference syncs on every inner iteration)
        for row in _native.stats_to_numpy(stats):
            print("\n".join(format_log(t, row)))
    if pose.data_ptr() != model_mean.data_ptr():
        model_mean.copy_(pose)  # the reference updates model_mean in place too (:84, :122)
    return pose
