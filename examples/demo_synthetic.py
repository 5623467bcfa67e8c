#!/usr/bin/env python
"""The reference's demo.py call pattern (pose_diffusion/demo.py:46-133) on the native path with synthetic inputs.

No checkpoint / DINO weights / hloc matches exist offline, so this script builds the model from the reference's config
dict (cfgs/default.yaml), keeps the random initialisation, feeds random images through the native multi-scale DINO ViT-S/16
extractor (or z ~ N(0,1) features with --no-images) and a geometry-consistent synthetic scene, and runs the sampler with and
without geometry-guided sampling, then the evaluation metrics of test.py against the synthetic ground truth.  With a real
checkpoint only one line changes: `model.load_state_dict(torch.load(ckpt), strict=True)`.
"""
import os
import sys
import time
from functools import partial

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import posediffusion_b200 as pdb
from posediffusion_b200 import synthetic as syn

MODEL_CFG = {  # cfgs/default.yaml:18-40
    "pose_encoding_type": "absT_quaR_logFL",
    "IMAGE_FEATURE_EXTRACTOR": {"_target_": "models.MultiScaleImageFeatureExtractor", "freeze": False},  # cfgs/default.yaml:20-22
    "DENOISER": {"_target_": "models.Denoiser",
                 "TRANSFORMER": {"_target_": "models.TransformerEncoderWrapper", "d_model": 512, "nhead": 4, "dim_feedforward": 1024,
                                 "num_encoder_layers": 8, "dropout": 0.1, "batch_first": True, "norm_first": True}},
    "DIFFUSER": {"_target_": "models.GaussianDiffusion", "beta_schedule": "custom"},
}
GGS_CFG = dict(syn.default_ggs_cfg(), verbose=False)  # cfgs/default.yaml:6-13


def main(frames: int = 20, matches_per_pair: int = 512, use_images: bool = True):
    from posediffusion_b200 import metric

    device = torch.device("cuda:0")
    model = pdb.PoseDiffusionModel(**MODEL_CFG).to(device).eval()
    torch.manual_seed(0)
    if use_images:  # demo.py:108 passes image=[B, N, 3, 224, 224]; features are computed once and reused below
        images = torch.rand(1, frames, 3, 224, 224, device=device)
        z = model(image=images, training=False)["z"]
    else:
        z = torch.randn(1, frames, 384, device=device)
    matches_dict, gt_pose, _ = syn.scene_matches(frames, matches_per_pair, seed=0, ordered=False)  # unordered pairs, like hloc
    cond_fn = partial(pdb.geometry_guided_sampling, matches_dict=matches_dict, GGS_cfg=GGS_CFG)
    for name, kwargs in (("GGS off", {}), ("GGS on", dict(cond_fn=cond_fn, cond_start_step=GGS_CFG["start_step"]))):
        model(z=z, training=False, **kwargs)  # warm-up (weight packing, match upload)
        torch.cuda.synchronize()
        start = time.time()
        pred = model(z=z, training=False, **kwargs)
        torch.cuda.synchronize()
        cams = pred["pred_cameras"]
        gt = pdb.pose_encoding_to_camera(torch.from_numpy(gt_pose).to(device).reshape(1, frames, 9))
        r_deg, t_deg = metric.camera_to_rel_deg(cams, gt, device, 1)  # test.py:217
        auc = metric.calculate_auc_np(r_deg.cpu().numpy(), t_deg.cpu().numpy(), max_threshold=30)
        print(f"{name:8s}: {time.time() - start:.4f} s for {frames} frames; R {tuple(cams.R.shape)}, T {tuple(cams.T.shape)}, "
              f"focal {cams.focal_length.mean().item():.3f}; vs synthetic GT (random weights): rel. rotation {r_deg.mean().item():.1f} deg, "
              f"AUC@30 {auc:.3f}")


if __name__ == "__main__":
    main(use_images="--no-images" not in sys.argv)
