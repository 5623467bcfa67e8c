"""Backbone training (csrc/api_vit_train.cu) at the sizes it runs, against the float64 autograd of oracle/vit_train_oracle.py on
the GPU.

Bound per tensor as in tests/test_gpu_vit_train.py: rel(gpu, f64) <= 5 rel(tf32 oracle, f64) + 1e-6 for z and each of the 150
gradients.  Covered here: every key-slot boundary of the attention backward (vit_attn_bwd_kernel keeps key j in lane slot
j = lane + 32m, m < 8: L = 2 ... 256), several scales in one call, upsampling, the position-table gradient (the adjoint of the
bicubic resampling) on one-cell, one-row and one-sided grids, 512 images at 224^2 against float64, the refusals, and the swap-AB
tensor-core tiles.
"""
import ctypes as C
import math

import pytest
import torch

from oracle import vit_train_oracle as vo
from oracle.vit_f64 import tokens_per_scale
from posediffusion_b200 import _native
from test_gpu_vit_train import DEFAULT, images, make_extractor, native_grads, rel

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")


def check(case, n, h, w, scales=(1,), allowance=0.0, chunk=None, seed=1):
    """z and the 150 gradients of n images against the chunked float64 oracle; `allowance` is added to the gradients' bound.
    Prints and returns the worst error / bound."""
    ext, state = make_extractor(scales=scales)
    img = images(n, h, w, seed)
    g = torch.randn(n, 384, generator=torch.Generator().manual_seed(7))
    z, grads = native_grads(ext, img, g)
    del ext
    chunk = chunk or n
    zr, ref = vo.features_and_grads_chunked(state, img, scales, g, chunk=chunk, device=DEV)
    zt, tf = vo.features_and_grads_chunked(state, img, scales, g, tf32=True, chunk=chunk, device=DEV)
    rows = [("z", z, zr, zt, 0.0)] + [(k, grads[k], ref[k], tf[k], allowance) for k in ref]
    worst, bad = (0.0, None), []
    for name, got, r, t_, extra in rows:
        assert torch.isfinite(got).all(), name
        d_tf, d = rel(t_.reshape(-1), r.reshape(-1)), rel(got.reshape(-1), r.reshape(-1))
        bound = 5 * d_tf + 1e-6 + extra
        worst = max(worst, (d / bound, f"{name}: {d:.2e} vs TF32 oracle {d_tf:.2e}"))
        if d > bound:
            bad.append((name, d, d_tf, bound))
    print(f"{case}: largest error / bound {worst[0]:.3f} ({worst[1]})")
    assert not bad, bad[:5]
    return worst[0]


ATT_CASES = [  # (h, w, scale factors): tokens per sequence
    (16, 16, (1,)),  # 2: a 1x1 grid
    (16, 496, (1,)),  # 32: a 1x31 grid, the last key of the first slot
    (64, 128, (1,)),  # 33: first key of the second slot
    (112, 144, (1,)),  # 64
    (64, 256, (1,)),  # 65: third slot
    (128, 192, (1,)),  # 97: fourth slot
    (128, 256, (1,)),  # 129: fifth slot
    (160, 256, (1,)),  # 161: sixth slot
    (224, 256, (1,)),  # 225: eighth slot
    (240, 272, (1,)),  # 256: the limit
    (240, 272, (1, 1 / 2, 1 / 3, 1 / 4)),  # 256, 57, 26, 13 in one call, at the scale limit
    (64, 64, (2,)),  # upsampled input: 65
]


@pytest.mark.parametrize("h,w,scales", ATT_CASES, ids=[f"{h}x{w}-L{'-'.join(map(str, tokens_per_scale(h, w, s)))}" for h, w, s in ATT_CASES])
def test_attention_lengths_against_oracle(h, w, scales):
    check(f"{h}x{w} L={tokens_per_scale(h, w, scales)}", 2, h, w, scales, seed=h + w)


@pytest.mark.parametrize("h,w,scales", [(256, 112, (1,)), (224, 239, (1,)), (448, 464, (1 / 2,))])
def test_position_gradient_of_resampled_grids(h, w, scales):
    """16x7 (upsampled in height, downsampled in width), 14x14 of a non-square image, 14x14 after halving 448x464."""
    check(f"position table {h}x{w} scales={scales}", 2, h, w, scales, seed=h * w)


def test_512_images_against_chunked_float64():
    """The released recipe's largest step (512 images of 224^2 at the default scales, 135 168 tokens) against float64 run in
    32-image chunks.  A dW element is one fp32 chain over all tokens: the bound adds 16 sqrt(S) 2^-24 (3.5e-4 here)."""
    S = 512 * sum(tokens_per_scale(224, 224, DEFAULT))
    check("512 images", 512, 224, 224, DEFAULT, allowance=16 * math.sqrt(S) * 2.0 ** -24, chunk=32, seed=9)


def test_refusals_launch_nothing_and_leave_the_context_usable():
    """257 tokens (256x256) and five scales: no workspace size, NativeError from the binding, PDB_ERR_LIMIT from the C entry
    point with a valid workspace, no kernel launched; a normal step afterwards gives the same bits as before."""
    ext, _ = make_extractor(scales=(1,))
    ctx = _native.Context.get(DEV)
    params = list(ext._net.parameters())
    img, g = images(2, 64, 64, 3), torch.randn(2, 384, generator=torch.Generator().manual_seed(4))
    z0, g0 = native_grads(ext, img, g)
    count = ctx.launch_count
    ws, z = torch.zeros(4096, device=DEV), torch.empty(1, 384, device=DEV)
    arr = (C.c_void_p * len(params))(*[C.c_void_p(q.data_ptr()) for q in params])
    for h, w, scales in ((256, 256, (1,)), (224, 224, (1, 1 / 2, 1 / 3, 1 / 4, 1 / 5))):
        im = images(1, h, w).to(DEV)
        assert _native.vit_train_workspace_bytes(1, h, w, scales) == 0
        with pytest.raises(_native.NativeError, match="unsupported backbone training shape"):
            ctx.vit_train_forward(params, im, scales)
        sf = (C.c_double * len(scales))(*scales)
        rc = ctx.lib.pdb_vit_train_forward(ctx.handle, arr, im.data_ptr(), 1, h, w, sf, len(scales), ws.data_ptr(), z.data_ptr(),
                                           _native._stream_ptr(DEV))
        assert rc == _native.PDB_ERR_LIMIT, (h, w, scales, rc)
    assert ctx.launch_count == count
    torch.cuda.synchronize()
    z1, g1 = native_grads(ext, img, g)
    assert torch.equal(z0, z1) and all(torch.equal(g0[k], g1[k]) for k in g0)


@pytest.mark.parametrize("n,h,w", [(1, 64, 64), (5, 16, 16)])
def test_swap_ab_tiles_against_oracle(n, h, w):
    """With the swap-AB switch on, GEMMs of at most 96 tokens with O % 128 == 0 run the swapped tiles (17 and 10 tokens)."""
    ctx = _native.Context.get(DEV)
    ctx.set_tc_swap(True)
    try:
        check(f"swap-AB {n}x{h}x{w}", n, h, w, seed=n + h)
    finally:
        ctx.set_tc_swap(False)
