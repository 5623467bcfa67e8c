"""wgmma + TMA linear layer (csrc/tc_linear.cuh) vs a plain PyTorch fp32 matmul of the same op.
Tolerance: TF32 products (10-bit mantissa), fp32 accumulate -> 2e-3 of max |y| (stated; K <= 1024)."""
import numpy as np
import pytest
import torch

from posediffusion_b200 import _native

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    assert torch.cuda.is_available()
    return _native.Context.get("cuda:0")


@pytest.fixture(params=[False, True], ids=["tiles128", "swapAB"])
def swap_on(ctx, request):
    ctx.set_tc_swap(request.param)
    yield request.param
    ctx.set_tc_swap(False)


# with swap_on, S <= 96 and O % 128 == 0 takes the swap-AB instantiation (weights on the wgmma M side, 32 / 64 / 96 tokens on the N side)
@pytest.mark.parametrize("S,O,K", [(128, 64, 32), (128, 512, 512), (160, 1536, 512), (20, 512, 1024), (300, 1024, 512), (1280, 512, 384),
                                   (5, 128, 512), (20, 1536, 512), (33, 512, 256), (64, 1024, 512), (80, 512, 1024), (96, 1536, 512),
                                   (20, 64, 512)])
@pytest.mark.parametrize("epi", ["plain", "bias_res_relu"])
def test_tc_linear_matches_fp32(ctx, S, O, K, epi, swap_on):
    g = torch.Generator(device="cuda").manual_seed(S + O + K)
    x = torch.randn(S, K, device="cuda", generator=g)
    w = torch.randn(O, K, device="cuda", generator=g) * 0.05
    bias = torch.randn(O, device="cuda", generator=g) if epi != "plain" else None
    res = torch.randn(S, O, device="cuda", generator=g) if epi != "plain" else None
    y = ctx.tc_linear(x, w, bias, res, relu=(epi != "plain"))
    torch.backends.cuda.matmul.allow_tf32 = False
    ref = x.double() @ w.double().T
    if bias is not None:
        ref = torch.relu(ref + bias.double() + res.double())
    err = (y.double() - ref).abs().max().item()
    scale = ref.abs().max().item()
    assert err <= 2e-3 * scale, (err, scale)
    # and it is really TF32-accurate, not garbage that happens to be small: correlation with the fp64 result
    assert torch.corrcoef(torch.stack([y.double().flatten(), ref.flatten()]))[0, 1].item() > 0.99999


@pytest.mark.parametrize("S,O,K", [(160, 512, 512), (160, 512, 1024), (130, 512, 512), (640, 512, 1024), (20, 512, 64), (300, 1024, 512)])
def test_tc_linear_in_place_residual_split_k(ctx, S, O, K):
    """The residual-stream update h += x @ w^T + b, Y aliasing the residual: with fewer tiles than SMs the launcher splits K over
    the idle SMs and the partial products are added to Y with vector reductions (csrc/api_tc.cu).  Same tolerance."""
    g = torch.Generator(device="cuda").manual_seed(S * 7 + O + K)
    x = torch.randn(S, K, device="cuda", generator=g)
    w = torch.randn(O, K, device="cuda", generator=g) * 0.05
    bias = torch.randn(O, device="cuda", generator=g)
    h = torch.randn(S, O, device="cuda", generator=g)
    ref = x.double() @ w.double().T + bias.double() + h.double()
    y = ctx.tc_linear(x, w, bias, h, in_place=True)
    assert y.data_ptr() == h.data_ptr()
    err = (y.double() - ref).abs().max().item()
    assert err <= 2e-3 * ref.abs().max().item(), err
    assert torch.corrcoef(torch.stack([y.double().flatten(), ref.flatten()]))[0, 1].item() > 0.99999


TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)


@pytest.mark.parametrize("B,N", [(8, 20), (1, 20), (2, 80), (1, 5), (1, 80), (3, 20), (7, 20), (32, 20), (50, 20)])
def test_tensor_core_denoiser_engine_vs_fp32_engine_and_oracle(ctx, B, N, swap_on):
    """The wgmma/TMA engine (TF32 products, LayerNorm folded into the GEMM epilogue) against the exact-fp32 engine
    and the CPU oracle on the same inputs.  Tolerance 5e-3 absolute on eps (values O(0.1..1))."""
    import posediffusion_b200 as pdb
    from oracle import pose_oracle as po
    from posediffusion_b200 import synthetic as syn

    state = syn.random_denoiser_state(5, 0.05)
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(state, strict=True)
    den = den.to("cuda")
    c = den.native_context()
    g = torch.Generator().manual_seed(B * 100 + N)
    x = torch.randn(B, N, 9, generator=g) * 1.5
    z = torch.randn(B, N, 384, generator=g)
    t = torch.full((B,), 23, dtype=torch.long)
    try:
        c.set_denoiser_engine("fp32")
        exact = den(x.cuda(), t.cuda(), z.cuda()).cpu()
        c.set_denoiser_engine("tf32")
        fast = den(x.cuda(), t.cuda(), z.cuda()).cpu()
    finally:
        c.set_denoiser_engine("auto")
    with torch.no_grad():
        want = po.build_denoiser(state)(x, t, z)
    assert (exact - want).abs().max().item() < 5e-5
    err = (fast - want).abs().max().item()
    assert err < 5e-3, err
    assert err > 0  # it really took the TF32 path
