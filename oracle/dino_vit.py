"""TEST INFRASTRUCTURE ONLY -- CPU restatement of the image backbone the reference pulls from torch.hub.

`models/image_feature_extractor.py:43` does `torch.hub.load("facebookresearch/dino:main", "dino_vits16")`: the network is a
THIRD-PARTY dependency that is not under /root/reference and is not pinned (branch `main`; no network here).  This file
restates the published algorithm of that repository's `vision_transformer.py` (`vit_small(patch_size=16)`):

  * patch embedding: Conv2d(3, 384, kernel 16, stride 16) -> tokens in (row, column) order, class token prepended;
  * position embedding [1, 197, 384], bicubically resampled for other resolutions with the `+0.1` scale-factor trick
    (`interpolate_pos_encoding`), i.e. `F.interpolate(..., scale_factor=((h//16 + 0.1)/14, (w//16 + 0.1)/14), mode="bicubic")`,
    applied here as the matrix that call is on the 196 grid cells (`resample_matrix`), so that autograd gives its transpose;
  * 12 pre-norm blocks: x += proj(MHSA(LN(x))), x += fc2(GELU(fc1(LN(x)))), 6 heads of 64, qkv with bias, LN eps 1e-6;
  * final LayerNorm, the class token is the feature (head = Identity).

Parity status: **unpinned against the original hub code** (absent); the block arithmetic is pinned instead against an
independent implementation of the same architecture, `transformers.ViTModel` (tests/test_features_cpu.py), and the
multi-scale wrapper around it is the reference's own `MultiScaleImageFeatureExtractor`, imported unmodified with
`torch.hub.load` redirected here (oracle/make_golden_features.py -> tests/golden/features.npz).  Parameter names follow the hub checkpoint
(`image_feature_extractor._net.*` in the released PoseDiffusion checkpoint) so a state_dict loads strictly.
"""
from __future__ import annotations

import functools
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

EMBED, DEPTH, HEADS, PATCH, MLP = 384, 12, 6, 16, 1536


GRID0 = 14  # the stored position grid


@functools.lru_cache(maxsize=None)
def resample_matrix(gh: int, gw: int) -> torch.Tensor:
    """R_s [gh*gw, 196], float64: interpolate_pos_encoding's bicubic resampling of the 14x14 grid at scale (grid + 0.1) / 14,
    row-major cells, read off F.interpolate on the CPU applied to the 196 basis grids.  The table is then a product, whose
    autograd is R_s^T.  Autograd through F.interpolate itself is not: when the grid keeps its 14x14 size (a non-square image)
    torch's bicubic backward copies the gradient through as if the resampling were the identity (9.5 % off R_s^T), and the CUDA
    forward copies the grid."""
    basis = torch.eye(GRID0 * GRID0, dtype=torch.float64).reshape(-1, 1, GRID0, GRID0)
    out = F.interpolate(basis, scale_factor=((gh + 0.1) / GRID0, (gw + 0.1) / GRID0), mode="bicubic")
    assert tuple(out.shape[-2:]) == (gh, gw)
    return out.reshape(GRID0 * GRID0, gh * gw).T.contiguous()


class _Attention(nn.Module):
    def __init__(self):
        super().__init__()
        self.qkv = nn.Linear(EMBED, 3 * EMBED, bias=True)
        self.proj = nn.Linear(EMBED, EMBED)

    def forward(self, x):
        B, L, C = x.shape
        qkv = self.qkv(x).reshape(B, L, 3, HEADS, C // HEADS).permute(2, 0, 3, 1, 4)
        q, k, v = qkv[0], qkv[1], qkv[2]
        att = (q @ k.transpose(-2, -1)) * (C // HEADS) ** -0.5
        att = att.softmax(dim=-1)
        return self.proj((att @ v).transpose(1, 2).reshape(B, L, C))


class _Mlp(nn.Module):
    def __init__(self):
        super().__init__()
        self.fc1 = nn.Linear(EMBED, MLP)
        self.fc2 = nn.Linear(MLP, EMBED)

    def forward(self, x):
        return self.fc2(F.gelu(self.fc1(x)))


class _Block(nn.Module):
    def __init__(self):
        super().__init__()
        self.norm1 = nn.LayerNorm(EMBED, eps=1e-6)
        self.attn = _Attention()
        self.norm2 = nn.LayerNorm(EMBED, eps=1e-6)
        self.mlp = _Mlp()

    def forward(self, x):
        x = x + self.attn(self.norm1(x))
        return x + self.mlp(self.norm2(x))


class _PatchEmbed(nn.Module):
    def __init__(self):
        super().__init__()
        self.proj = nn.Conv2d(3, EMBED, kernel_size=PATCH, stride=PATCH)

    def forward(self, x):
        return self.proj(x).flatten(2).transpose(1, 2)


class DinoViTSmall16(nn.Module):
    def __init__(self):
        super().__init__()
        self.cls_token = nn.Parameter(torch.zeros(1, 1, EMBED))
        self.pos_embed = nn.Parameter(torch.zeros(1, 1 + (224 // PATCH) ** 2, EMBED))
        self.patch_embed = _PatchEmbed()
        self.blocks = nn.ModuleList([_Block() for _ in range(DEPTH)])
        self.norm = nn.LayerNorm(EMBED, eps=1e-6)
        nn.init.trunc_normal_(self.pos_embed, std=0.02)
        nn.init.trunc_normal_(self.cls_token, std=0.02)
        for m in self.modules():
            if isinstance(m, nn.Linear):
                nn.init.trunc_normal_(m.weight, std=0.02)
                nn.init.zeros_(m.bias)

    def interpolate_pos_encoding(self, n_patches: int, h: int, w: int):
        n0 = self.pos_embed.shape[1] - 1
        if n_patches == n0 and w == h:
            return self.pos_embed
        assert n0 == GRID0 * GRID0, n0
        R = resample_matrix(h // PATCH, w // PATCH).to(self.pos_embed.device, self.pos_embed.dtype)
        return torch.cat((self.pos_embed[:, :1], (R @ self.pos_embed[0, 1:])[None]), dim=1)

    def prepare_tokens(self, img):
        B, _, h, w = img.shape
        x = self.patch_embed(img)
        x = torch.cat((self.cls_token.expand(B, -1, -1), x), dim=1)
        return x + self.interpolate_pos_encoding(x.shape[1] - 1, h, w)

    def forward(self, img, return_tokens: bool = False):
        x = self.prepare_tokens(img)
        stages = [x]
        for blk in self.blocks:
            x = blk(x)
            stages.append(x)
        x = self.norm(x)
        return (x[:, 0], stages) if return_tokens else x[:, 0]


def randomize(net: DinoViTSmall16, seed: int, qkv_std: float = 0.08) -> DinoViTSmall16:
    """Deterministic non-trivial parameters for parity tests: non-zero biases, non-unit LayerNorm affine and sharper
    attention logits than the 0.02 init gives (so key indexing / softmax-scale mistakes are visible)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for name, p in net.named_parameters():
            if name.endswith("qkv.weight"):
                p.copy_(torch.randn(p.shape, generator=g) * qkv_std)
            elif name.endswith("norm1.weight") or name.endswith("norm2.weight") or name == "norm.weight":
                p.copy_(1.0 + 0.1 * torch.randn(p.shape, generator=g))
            elif name.endswith(".bias"):
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            elif name in ("cls_token", "pos_embed"):
                p.copy_(0.05 * torch.randn(p.shape, generator=g))
            else:
                fan_in = p[0].numel()
                p.copy_(torch.randn(p.shape, generator=g) * (0.7 / math.sqrt(fan_in)))
    return net


RESNET_MEAN = (0.485, 0.456, 0.406)
RESNET_STD = (0.229, 0.224, 0.225)


def multiscale_features(net: DinoViTSmall16, image_rgb: torch.Tensor, scale_factors, return_stages: bool = False):
    """MultiScaleImageFeatureExtractor.forward restated (models/image_feature_extractor.py:63-87): ResNet normalisation, the
    backbone at every scale (bilinear, align_corners=False), features summed in order and divided by the number of scales.
    With return_stages also, per scale, the residual stream after prepare_tokens and after every block (the probes the CUDA
    path's debug dump is compared with).  Pinned against the reference's own wrapper by tests/golden/features.npz."""
    if len(scale_factors) <= 0:
        raise ValueError(f"Wrong format of self.scale_factors: {scale_factors}")
    mean = torch.tensor(RESNET_MEAN).view(1, 3, 1, 1)
    std = torch.tensor(RESNET_STD).view(1, 3, 1, 1)
    normed = (image_rgb - mean) / std
    total, stages = None, []
    for f in scale_factors:
        inp = normed if f == 1 else F.interpolate(normed, scale_factor=f, mode="bilinear", align_corners=False)
        feat, st = net(inp, return_tokens=True)
        stages.append(st)
        total = feat if total is None else total + feat
    z = total / len(scale_factors)
    return (z, stages) if return_stages else z
