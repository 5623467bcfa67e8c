"""Denoiser training (csrc/api_train.cu) at the sizes it runs, against the float64 oracle (oracle/train_oracle.py) on the GPU.

Bound per tensor, as in tests/test_gpu_train.py: rel(gpu, f64) <= 5 rel(tf32 oracle, f64) + 1e-6, with rel the relative L2
distance of the whole tensor; dL/dz is bounded the same way.  Covered here:
  - every frame count where the attention kernels change shape: N = 1, 2, the key-slot boundary 31 / 32 / 33 (key j sits in
    lane slot j = lane + 32m, m < 2) and the shared-memory limit 63 / 64, with and without dropout; 65 refused;
  - the released recipe's step, three sequence shapes x batch_repeat 90 (about 46 000 tokens): every forward projection and every
    dX GEMM on the 128-feature tensor-core tiles, every dW one fp32 chain over all tokens.  Row-wise and per-sequence outputs are
    bit-identical to the same sequences run in chunks of at most 1 280 tokens (64-feature tiles);
  - the swap-AB tensor-core tiles (at most 96 tokens) switched on.
"""
import ctypes as C
import math

import pytest
import torch

from oracle import train_oracle as to
from posediffusion_b200 import _native
from posediffusion_b200 import synthetic as syn
from test_gpu_train import NAMES, make_diffuser, rel

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
RELEASED = [(51, 10), (10, 50), (170, 3)]  # distinct sequences x frames (tools/train_step_time.py), each repeated 90 times
REPEAT = 90
CHUNK_TOKENS = 1280  # qkv at 1 280 tokens: 12 x 10 = 120 128-feature tiles, fewer than the H100's 132 SMs
ORACLE_TOKENS = 4096  # float64 oracle chunk on the GPU


def inputs(B, N, seed, distinct=None):
    """x_start, t, noise, z, grad_loss, grad_x0.  With `distinct`, z holds the features of `distinct` sequences repeated
    B / distinct times (z.repeat, as PoseDiffusionModel does for batch_repeat); poses, timesteps and noise are all distinct."""
    g = torch.Generator().manual_seed(500 + seed)
    x = torch.randn(B, N, 9, generator=g) * 0.5
    noise = torch.randn(B, N, 9, generator=g)
    t = torch.randint(0, 100, (B,), generator=g)
    gl, gx = torch.randn(B, N, 9, generator=g), torch.randn(B, N, 9, generator=g)
    d = distinct or B
    z = syn.random_features(d, N, seed).repeat(B // d, 1, 1)
    return x, t, noise, z, gl, gx


def native(dif, x, t, noise, z, gl, gx, p=0.0, seed=0, want_grads=True):
    """One native step with dL/dz: ({loss, x_0_pred, x_t, dz} on the device, {name: gradient} or None)."""
    den = dif.model
    den.zero_grad(set_to_none=True)
    zd = z.to(DEV).requires_grad_(True)
    loss, x0, x_t = den.train_step_forward(x.to(DEV), t.to(DEV), noise.to(DEV), zd, p, seed, dif.loss_type)
    torch.autograd.backward([loss, x0], [gl.to(DEV), gx.to(DEV)])
    out = {"loss": loss.detach(), "x_0_pred": x0.detach(), "x_t": x_t.detach(), "dz": zd.grad}
    grads = {n: q.grad.clone() for n, q in den.named_parameters()} if want_grads else None
    den.zero_grad(set_to_none=True)
    return out, grads


def check(case, state, args, out, grads, p=0.0, seed=None, offset=0, allowance=0.0, keys=("x_t", "x_0_pred", "loss")):
    """Outputs `keys`, dz and (unless grads is None) the 108 gradients against the chunked float64 oracle; `allowance` is added
    to the bound of dz and the gradients.  Prints and returns the worst error / bound."""
    N = args[0].shape[1]
    kw = dict(p=p, seed=seed, chunk=max(1, ORACLE_TOKENS // N), device=DEV, offset=offset)
    ref, rg, rdz = to.loss_and_grads_chunked(state, *args, "l1", **kw)
    tf, tg, tdz = to.loss_and_grads_chunked(state, *args, "l1", tf32="trunc", **kw)
    rows = [(k, out[k], ref[k], tf[k], 0.0) for k in keys] + [("dz", out["dz"], rdz, tdz, allowance)]
    if grads is not None:
        rows += [(n, grads[n], rg[n], tg[n], allowance) for n in NAMES]
    worst, bad = (0.0, None), []
    for name, got, r, t_, extra in rows:
        d_tf, d = rel(t_, r), rel(got, r)
        bound = 5 * d_tf + 1e-6 + extra
        worst = max(worst, (d / bound, f"{name}: {d:.2e} vs TF32 oracle {d_tf:.2e}"))
        if d > bound:
            bad.append((name, d, d_tf, bound))
    print(f"{case}: largest error / bound {worst[0]:.3f} ({worst[1]})")
    assert not bad, bad[:5]
    return worst[0]


# ---- frame counts --------------------------------------------------------------------------------------------------------
# B x N is not a multiple of 32 (the padded token count Sp differs from S) except at N = 32 and 64, where no B gives one.  N = 1
# runs 21 sequences: at 5 tokens a weight gradient is a sum of 5 rows, and one ReLU input that fp32 arithmetic puts on the other
# side of zero than the float64 TF32 emulation does (an fp32 evaluation of the same TF32 operands on the CPU shows it, 15.6x the
# bound on layers.2.linear1.bias) dominates the tensor's relative error.
FRAMES = [(21, 1), (3, 2), (3, 31), (3, 32), (3, 33), (3, 63), (3, 64)]


@pytest.mark.parametrize("p", [0.0, 0.1])
@pytest.mark.parametrize("B,N", FRAMES, ids=[f"N{n}" for _, n in FRAMES])
def test_frame_counts_against_oracle(B, N, p):
    dif, state = make_diffuser()
    args = inputs(B, N, N)
    seed = 0x5EED_0000 + N
    out, grads = native(dif, *args, p=p, seed=seed)
    check(f"B={B} N={N} p={p}", state, args, out, grads, p=p, seed=seed)


def test_65_frames_are_refused_before_any_launch():
    dif, _ = make_diffuser()
    ctx = _native.Context.get(DEV)
    small = inputs(3, 7, 1)
    before, gb = native(dif, *small)
    assert _native.train_workspace_bytes(1, 65) == 0
    x, t, noise, z, _, _ = (v.to(DEV) for v in inputs(1, 65, 2))
    count = ctx.launch_count
    with pytest.raises(_native.NativeError, match="at most 64 frames"):
        dif.p_losses(x, t, z, noise)
    params = dif.model.ordered_parameters()
    with pytest.raises(_native.NativeError, match="at most 64 frames"):
        ctx.train_forward(params, x, t.int(), noise, z, 0.0, 0, "l1")
    # the C entry point itself, with a valid workspace pointer: refused with PDB_ERR_LIMIT
    ws = torch.zeros(4096, device=DEV)
    loss, x_t, x0 = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
    t32 = t.int().contiguous()
    arr = (C.c_void_p * len(params))(*[C.c_void_p(q.data_ptr()) for q in params])
    rc = ctx.lib.pdb_train_forward(ctx.handle, arr, x.data_ptr(), t32.data_ptr(), noise.data_ptr(), z.data_ptr(), 1, 65, 0.0, 0, 0,
                                   ws.data_ptr(), loss.data_ptr(), x_t.data_ptr(), x0.data_ptr(), _native._stream_ptr(DEV))
    assert rc == _native.PDB_ERR_LIMIT
    assert ctx.launch_count == count
    torch.cuda.synchronize()
    after, ga = native(dif, *small)
    assert all(torch.equal(before[k], after[k]) for k in before)
    assert all(torch.equal(gb[n], ga[n]) for n in gb)


# ---- the released step ---------------------------------------------------------------------------------------------------
def released(distinct, N, seed):
    return inputs(distinct * REPEAT, N, seed, distinct)


@pytest.fixture(scope="module")
def tile_regimes():
    """The full-size step runs the 128-feature tiles and its chunks the 64-feature tiles (csrc/api_tc.cu: 128-feature tiles when
    O % 128 == 0 and (O / 128) * ceil(S / 128) >= SMs)."""
    sm = torch.cuda.get_device_properties(DEV).multi_processor_count
    smallest = min(d * REPEAT * n for d, n in RELEASED)
    assert (128 // 128) * math.ceil(smallest / 128) >= sm, sm  # _last.0 (128 features), the narrowest 128-divisible GEMM
    assert (1536 // 128) * math.ceil(CHUNK_TOKENS / 128) < sm, sm  # qkv, the widest GEMM
    return sm


@pytest.mark.parametrize("distinct,N", RELEASED, ids=[f"{d}x{n}x{REPEAT}" for d, n in RELEASED])
def test_released_step_without_dropout(tile_regimes, distinct, N):
    """Bit-identical twice and to 1 280-token chunks (loss, x_0_pred, x_t, dz); gradients and dz against the float64 oracle with
    a serial-accumulation allowance: a dW element is one fp32 chain over Sp tokens, 16 sqrt(Sp) 2^-24 (about 2e-4 at 45 920)."""
    dif, state = make_diffuser()
    args = released(distinct, N, N)
    B = args[0].shape[0]
    full, grads = native(dif, *args)
    again, grads2 = native(dif, *args)
    for k in full:
        assert torch.equal(full[k], again[k]), k
    for n in grads:
        assert torch.equal(grads[n], grads2[n]), n
    del again, grads2
    c = CHUNK_TOKENS // N
    for b0 in range(0, B, c):
        sl = slice(b0, b0 + c)
        part, _ = native(dif, *(a[sl] for a in args), want_grads=False)
        for k in part:
            assert torch.equal(part[k], full[k][sl]), (k, b0)
    Sp = (B * N + 31) // 32 * 32
    check(f"released {distinct}x{N}x{REPEAT} ({B * N} tokens) p=0", state, args, full, grads,
          allowance=16 * math.sqrt(Sp) * 2.0 ** -24)


@pytest.mark.parametrize("distinct,N", RELEASED, ids=[f"{d}x{n}x{REPEAT}" for d, n in RELEASED])
def test_released_step_with_dropout(tile_regimes, distinct, N):
    """p = 0.1: the first chunk's sequences are bit-identical to that chunk run alone with the same seed (the mask index is the
    flat element index, the same at offset 0); the last 8 sequences' loss, x_0_pred and dz against the oracle with the masks at
    their offsets."""
    dif, state = make_diffuser()
    args = released(distinct, N, N + 1)
    B = args[0].shape[0]
    seed = 0x1234_5678_9ABC + N
    full, _ = native(dif, *args, p=0.1, seed=seed, want_grads=False)
    c = CHUNK_TOKENS // N
    part, _ = native(dif, *(a[:c] for a in args), p=0.1, seed=seed, want_grads=False)
    for k in part:
        assert torch.equal(part[k], full[k][:c]), k
    last = {k: v[B - 8:] for k, v in full.items()}
    check(f"released {distinct}x{N}x{REPEAT} p=0.1, last 8 sequences", state, tuple(a[B - 8:] for a in args), last, None,
          p=0.1, seed=seed, offset=B - 8, keys=("x_0_pred", "loss"))


# ---- swap-AB tiles -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("B,N", [(2, 5), (4, 20)])
def test_swap_ab_tiles_against_oracle(B, N):
    """With the swap-AB switch on, every GEMM with at most 96 tokens and O % 128 == 0 runs the swapped tiles."""
    dif, state = make_diffuser()
    ctx = _native.Context.get(DEV)
    args = inputs(B, N, 70 + N)
    ctx.set_tc_swap(True)
    try:
        out, grads = native(dif, *args)
    finally:
        ctx.set_tc_swap(False)
    check(f"swap-AB B={B} N={N}", state, args, out, grads)
