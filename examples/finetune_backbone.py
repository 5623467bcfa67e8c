#!/usr/bin/env python
"""Five AdamW steps of the released training recipe's model (`IMAGE_FEATURE_EXTRACTOR.freeze: False`) on synthetic images and
cameras: the backbone and the denoiser train together, every gradient comes from the native sm_90a kernels.

    python examples/finetune_backbone.py
"""
import os
import sys
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import posediffusion_b200 as pdb  # noqa: E402

dev = torch.device("cuda:0")
transformer = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
model = pdb.PoseDiffusionModel(
    pose_encoding_type="absT_quaR_logFL",
    IMAGE_FEATURE_EXTRACTOR=dict(_target_="models.MultiScaleImageFeatureExtractor", freeze=False),
    DIFFUSER=dict(_target_="models.GaussianDiffusion", beta_schedule="custom"),
    DENOISER=dict(_target_="models.Denoiser", TRANSFORMER=transformer, target_dim=9, pivot_cam_onehot=True, z_dim=384, mlp_hidden_dim=128),
).to(dev).train()
sequences, frames, batch_repeat = 2, 5, 4
torch.manual_seed(0)
image = torch.rand(sequences, frames, 3, 224, 224, device=dev)
count = sequences * batch_repeat * frames
cameras = SimpleNamespace(R=torch.eye(3, device=dev).expand(count, 3, 3).contiguous(), T=torch.randn(count, 3, device=dev),
                          focal_length=1.5 + torch.rand(count, 2, device=dev))
optimizer = torch.optim.AdamW(model.parameters(), lr=1e-4)
for step in range(5):
    optimizer.zero_grad(set_to_none=True)
    loss = model(image=image, gt_cameras=cameras, training=True, batch_repeat=batch_repeat)["loss"].mean()
    loss.backward()
    optimizer.step()
    print(f"step {step}: loss {loss.item():.4f}")
