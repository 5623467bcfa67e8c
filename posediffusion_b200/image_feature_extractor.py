"""`MultiScaleImageFeatureExtractor` with the reference's constructor / forward (models/image_feature_extractor.py:27-87).

The backbone the reference downloads with `torch.hub.load("facebookresearch/dino:main", "dino_vits16")` is represented here by
`DinoViTSmall16`, a parameter container with the hub checkpoint's names and shapes (so the released checkpoint's
`image_feature_extractor._net.*` keys load strictly).  It has no PyTorch forward: features come from the native library
(pdb_extract_features -- patch embedding, the 12 blocks and the head as wgmma/TMA GEMMs + shared-memory attention).

With `freeze=False` (the released training recipe) and grad enabled, the forward runs the training path instead
(pdb_vit_train_forward / pdb_vit_backward through `_BackboneFeatures`): explicit LayerNorm, activations saved in a workspace the
autograd node owns, gradients into all 150 backbone tensors.
"""
from __future__ import annotations

from typing import List, Sequence

import torch
import torch.nn as nn

from . import _native

_EMBED, _DEPTH, _MLP, _PATCH = 384, 12, 1536, 16


class _Attn(nn.Module):
    def __init__(self):
        super().__init__()
        self.qkv = nn.Linear(_EMBED, 3 * _EMBED, bias=True)
        self.proj = nn.Linear(_EMBED, _EMBED)


class _Mlp(nn.Module):
    def __init__(self):
        super().__init__()
        self.fc1 = nn.Linear(_EMBED, _MLP)
        self.fc2 = nn.Linear(_MLP, _EMBED)


class _Block(nn.Module):
    def __init__(self):
        super().__init__()
        self.norm1 = nn.LayerNorm(_EMBED, eps=1e-6)
        self.attn = _Attn()
        self.norm2 = nn.LayerNorm(_EMBED, eps=1e-6)
        self.mlp = _Mlp()


class _PatchEmbed(nn.Module):
    def __init__(self):
        super().__init__()
        self.proj = nn.Conv2d(3, _EMBED, kernel_size=_PATCH, stride=_PATCH)


class DinoViTSmall16(nn.Module):
    """Parameters of dino `vit_small(patch_size=16)` in checkpoint order; compute is native."""

    def __init__(self):
        super().__init__()
        self.cls_token = nn.Parameter(torch.zeros(1, 1, _EMBED))
        self.pos_embed = nn.Parameter(torch.zeros(1, 1 + (224 // _PATCH) ** 2, _EMBED))
        self.patch_embed = _PatchEmbed()
        self.blocks = nn.ModuleList([_Block() for _ in range(_DEPTH)])
        self.norm = nn.LayerNorm(_EMBED, eps=1e-6)
        nn.init.trunc_normal_(self.pos_embed, std=0.02)
        nn.init.trunc_normal_(self.cls_token, std=0.02)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                nn.init.zeros_(m.bias)

    def forward(self, *args, **kwargs):
        raise RuntimeError("DinoViTSmall16 holds parameters only; call MultiScaleImageFeatureExtractor (native CUDA path)")


class _BackboneFeatures(torch.autograd.Function):
    """Native backbone forward whose activations live in a workspace tensor this graph node owns; backward (pdb_vit_backward)
    returns the gradients of the 150 parameters (none for the images).  The parameters are saved for backward, so changing one
    in place between the two raises torch's version error."""

    @staticmethod
    def forward(fctx, ctx, images, scale_factors, *params):
        ws, z = ctx.vit_train_forward(params, images, scale_factors)
        fctx.native, fctx.ws = ctx, ws
        fctx.save_for_backward(*params)
        return z

    @staticmethod
    def backward(fctx, grad_z):
        params = fctx.saved_tensors
        if fctx.ws is None:
            raise RuntimeError("the native training graph was already backpropagated and its workspace released")
        grads = fctx.native.vit_backward(params, fctx.ws, grad_z.contiguous().float())
        fctx.ws = None
        return (None, None, None, *grads)


class MultiScaleImageFeatureExtractor(nn.Module):
    def __init__(self, modelname: str = "dino_vits16", freeze: bool = False, scale_factors: Sequence[float] = (1, 1 / 2, 1 / 3)):
        super().__init__()
        self.freeze = freeze
        self.scale_factors: List[float] = list(scale_factors)
        if modelname != "dino_vits16":
            if "res" in modelname or "dino" in modelname:
                raise NotImplementedError(f"{modelname}: only dino_vits16 (cfgs/default.yaml) has a native backbone")
            raise ValueError(f"Unknown model name {modelname}")  # image_feature_extractor.py:46-47
        self._net = DinoViTSmall16()
        self._output_dim = self._net.norm.weight.shape[0]
        if self.freeze:
            for param in self.parameters():
                param.requires_grad = False

    def get_output_dim(self):
        return self._output_dim

    def _sync_weights(self, ctx: "_native.Context"):
        params = list(self._net.state_dict().values())
        if not hasattr(self, "_native_token"):
            self._native_token = _native.module_token()  # never reused, unlike id()
        key = (self._native_token,) + tuple((p.data_ptr(), p._version) for p in params)
        if getattr(ctx, "vit_key", None) != key:  # the context holds ONE backbone: reload if another module used it since
            ctx.load_vit(params)
            ctx.vit_key = key

    def forward(self, image_rgb: torch.Tensor) -> torch.Tensor:
        if len(self.scale_factors) <= 0:
            raise ValueError(f"Wrong format of self.scale_factors: {self.scale_factors}")  # :75-76
        if not image_rgb.is_cuda:
            raise _native.NativeError("image_rgb must be a CUDA tensor (posediffusion_b200 has no CPU fallback)")
        ctx = _native.Context.get(image_rgb.device)
        images = image_rgb.detach().to(torch.float32).contiguous()
        params = list(self._net.parameters())  # registration order = hub state_dict order (the module has no buffers)
        if torch.is_grad_enabled() and any(p.requires_grad for p in params):
            return _BackboneFeatures.apply(ctx, images, tuple(self.scale_factors), *params)
        with torch.no_grad():
            self._sync_weights(ctx)
            return ctx.extract_features(images, self.scale_factors)
