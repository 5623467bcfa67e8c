"""Float64 evaluation of the image feature extractor -- TEST INFRASTRUCTURE.

The network of oracle/dino_vit.py and the pyramid of `multiscale_features`, restated over plain tensors so that one block can
be applied to a given residual stream (teacher forcing on the device's debug dumps) and so that the operands can be rounded
the way pdb_extract_features reads them.  `mode`:

  None      exact, in the evaluator's dtype (float64; float32 reproduces `multiscale_features`);
  "tf32"    what the device computes, in float64: every GEMM operand truncated to TF32 (`train_oracle.tf32_round(.., "trunc")`,
            the tensor cores truncate); qkv and fc1 in the folded form of csrc/fold_ln.cuh, W' = fp32(W * gamma) truncated,
            colsum = sum_k W' and b' = b + W beta from the fp32 W' and W, epilogue rstd * (acc - mean * colsum) + b' on the raw
            stream; attention operands Q * 0.125, K, V and the unnormalised P rounded to nearest (the kernel's cvt.rna);
  "tf32_ln" the same roundings with LayerNorm applied explicitly before qkv / fc1 (what folding costs, measured against "tf32").

The device tests bound |device - float64| by four times |"tf32" run - float64| per token row (DESIGN.md section 4.6).
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence

import torch
import torch.nn.functional as F

from oracle.dino_vit import EMBED, HEADS, PATCH, RESNET_MEAN, RESNET_STD, resample_matrix
from oracle.train_oracle import tf32_round

GRID0 = 14
MODES = (None, "tf32", "tf32_ln")


def _trunc(x):
    return tf32_round(x, "trunc")


def _rna(x):
    return tf32_round(x, "rn")


class VitF64:
    """Evaluator over one DinoViTSmall16 state_dict (hub parameter names), on `device` (default the CPU)."""

    def __init__(self, state: Dict[str, torch.Tensor], dtype: torch.dtype = torch.float64, device="cpu"):
        self.dtype = dtype
        self.device = torch.device(device)
        self.p = {k: v.detach().to(device, dtype) for k, v in state.items()}
        p32 = {k: v.detach().to(device, torch.float32) for k, v in state.items()}
        self.folded = {}  # (block, "qkv" | "fc1") -> (W', colsum, b') as the device holds them, widened
        for l in range(12):
            pre = f"blocks.{l}."
            for which, lin, norm in (("qkv", "attn.qkv", "norm1"), ("fc1", "mlp.fc1", "norm2")):
                w, b = p32[pre + lin + ".weight"], p32[pre + lin + ".bias"]
                wf = w * p32[pre + norm + ".weight"]  # fp32 product, as fold_ln_kernel stores it
                self.folded[(l, which)] = (wf.to(dtype), wf.to(dtype).sum(1), b.to(dtype) + w.to(dtype) @ p32[pre + norm + ".bias"].to(dtype))

    # ---- pieces --------------------------------------------------------------------------------------------------------
    def linear(self, x, w, b, mode):
        if mode is None:
            return x @ w.T + b
        return _trunc(x) @ _trunc(w).T + b

    def ln_linear(self, x, l: int, which: str, mode):
        """LayerNorm (norm1 before qkv, norm2 before fc1) followed by the projection, in block l (0-based)."""
        pre = f"blocks.{l}."
        lin, norm = ("attn.qkv", "norm1") if which == "qkv" else ("mlp.fc1", "norm2")
        if mode == "tf32":
            wf, colsum, bf = self.folded[(l, which)]
            mean = x.mean(-1, keepdim=True)
            rstd = ((x - mean).pow(2).mean(-1, keepdim=True) + 1e-6).rsqrt()
            return rstd * (_trunc(x) @ _trunc(wf).T - mean * colsum) + bf
        y = F.layer_norm(x, (EMBED,), self.p[pre + norm + ".weight"], self.p[pre + norm + ".bias"], 1e-6)
        return self.linear(y, self.p[pre + lin + ".weight"], self.p[pre + lin + ".bias"], mode)

    def attention(self, qkv, mode):
        B, L, _ = qkv.shape
        q, k, v = qkv.reshape(B, L, 3, HEADS, EMBED // HEADS).permute(2, 0, 3, 1, 4)
        if mode is None:
            att = ((q @ k.transpose(-2, -1)) * (EMBED // HEADS) ** -0.5).softmax(dim=-1) @ v
        else:
            s = _rna(q * 0.125) @ _rna(k).transpose(-2, -1)
            p = (s - s.amax(-1, keepdim=True)).exp()
            att = (_rna(p) @ _rna(v)) / p.sum(-1, keepdim=True)
        return att.transpose(1, 2).reshape(B, L, EMBED)

    def block(self, k: int, x: torch.Tensor, mode=None) -> torch.Tensor:
        """Block k (1-based, the debug_stage numbering) applied to the residual stream x [n, L, 384]."""
        l, pre, P = k - 1, f"blocks.{k - 1}.", self.p
        x = x.to(self.dtype)
        x = x + self.linear(self.attention(self.ln_linear(x, l, "qkv", mode), mode), P[pre + "attn.proj.weight"], P[pre + "attn.proj.bias"], mode)
        h = F.gelu(self.ln_linear(x, l, "fc1", mode))
        return x + self.linear(h, P[pre + "mlp.fc2.weight"], P[pre + "mlp.fc2.bias"], mode)

    def pos_table(self, gh: int, gw: int, h: int, w: int) -> torch.Tensor:
        """interpolate_pos_encoding: the stored table for 196 patches of a square (h == w pixels) input, else bicubic with
        scale (grid + 0.1) / 14.  [1 + gh*gw, 384]."""
        pos = self.p["pos_embed"][0]
        if gh * gw == GRID0 * GRID0 and h == w:
            return pos
        R = resample_matrix(gh, gw).to(pos.device, pos.dtype)
        return torch.cat([pos[:1], R @ pos[1:]])

    def pyramid(self, image_rgb: torch.Tensor, scale_factors: Sequence[float]) -> List[torch.Tensor]:
        mean = torch.tensor(RESNET_MEAN, dtype=self.dtype, device=self.device).view(1, 3, 1, 1)
        std = torch.tensor(RESNET_STD, dtype=self.dtype, device=self.device).view(1, 3, 1, 1)
        normed = (image_rgb.to(self.device, self.dtype) - mean) / std
        return [normed if f == 1 else F.interpolate(normed, scale_factor=f, mode="bilinear", align_corners=False) for f in scale_factors]

    def prepare_tokens(self, img: torch.Tensor, mode=None) -> torch.Tensor:
        """Stage 0 of one scale: patch GEMM, class token, position table.  img [n,3,h,w] normalised -> [n, 1 + gh*gw, 384]."""
        n, _, h, w = img.shape
        gh, gw = h // PATCH, w // PATCH
        patches = img[:, :, :gh * PATCH, :gw * PATCH].reshape(n, 3, gh, PATCH, gw, PATCH).permute(0, 2, 4, 1, 3, 5).reshape(n, gh * gw, -1)
        tok = self.linear(patches, self.p["patch_embed.proj.weight"].reshape(EMBED, -1), self.p["patch_embed.proj.bias"], mode)
        x = torch.cat([self.p["cls_token"].expand(n, 1, EMBED), tok], dim=1)
        return x + self.pos_table(gh, gw, h, w)

    def features(self, image_rgb: torch.Tensor, scale_factors: Sequence[float], mode=None, return_stages: bool = False):
        """multiscale_features: z [n,384] (and, per scale, the 13 residual streams [n, L, 384] after stage 0..12)."""
        if len(scale_factors) <= 0:
            raise ValueError(f"Wrong format of self.scale_factors: {scale_factors}")
        total, stages = None, []
        for img in self.pyramid(image_rgb, scale_factors):
            x = self.prepare_tokens(img, mode)
            st = [x]
            for k in range(1, 13):
                x = self.block(k, x, mode)
                st.append(x)
            stages.append(st)
            feat = F.layer_norm(x[:, 0], (EMBED,), self.p["norm.weight"], self.p["norm.bias"], 1e-6)
            total = feat if total is None else total + feat
        z = total / len(scale_factors)
        return (z, stages) if return_stages else z


def tokens_per_scale(h: int, w: int, scale_factors: Sequence[float]) -> List[int]:
    """1 + gh*gw per scale, with F.interpolate's output size floor(size * f) (what pdb_extract_features computes)."""
    out = []
    for f in scale_factors:
        oh, ow = (h, w) if f == 1 else (int(h * float(f) // 1), int(w * float(f) // 1))
        out.append(1 + (oh // PATCH) * (ow // PATCH))
    return out


def split_rows(rows: torch.Tensor, n: int, tokens: Sequence[int]) -> List[torch.Tensor]:
    """The device's debug dump [sum_s n*L_s, 384] (scale-major, image, token) -> per scale [n, L_s, 384]."""
    out, r = [], 0
    for L in tokens:
        out.append(rows[r:r + n * L].reshape(n, L, EMBED))
        r += n * L
    assert r == rows.shape[0], (r, rows.shape)
    return out


def join_rows(per_scale: Sequence[torch.Tensor]) -> torch.Tensor:
    return torch.cat([x.reshape(-1, EMBED) for x in per_scale])
