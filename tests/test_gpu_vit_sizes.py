"""The image feature extractor (pdb_extract_features, csrc/api_vit.cu) at the sizes it runs: the frame counts of the demo and the
evaluation on both tensor-core tile widths of every ViT GEMM, a training step's 512 images, every attention-length boundary,
position tables of non-square inputs, rows whose mean dominates the folded LayerNorm, and the swap-AB tiles.

The arbiter is oracle/vit_f64.py.  Per token row (per image for z) the device must satisfy
    |dev - f64| <= 4 |tf32 - f64| + 1e-6 |ref|
where tf32 is the float64 run with the device's operand roundings and ref is the float64 value; for a block stage, ref is the
block's update X_k - X_{k-1}, and the block is teacher-forced on the device's own stage k-1 (one block's error in isolation).
DESIGN.md section 4.6 lists the largest error/bound ratios measured per case."""
import math

import pytest
import torch

from oracle.dino_vit import DinoViTSmall16, randomize
from oracle.make_golden_features import VIT_SEED, images_for
from oracle.vit_f64 import VitF64, join_rows, split_rows, tokens_per_scale
from posediffusion_b200 import _native

pytestmark = pytest.mark.gpu
SF = [1, 1 / 2, 1 / 3]
TOKENS = sum(tokens_per_scale(224, 224, SF))  # 264 rows per 224^2 image at the default scales
GEMMS = {"patch/proj/fc2": 384, "qkv": 1152, "fc1": 1536}
RATIOS = {}


@pytest.fixture(scope="module", autouse=True)
def report():
    yield
    print("\nlargest error/bound ratio per case:")
    for case, r in sorted(RATIOS.items()):
        print(f"  {case}: {r:.3f}")


@pytest.fixture(scope="module")
def state():
    return randomize(DinoViTSmall16(), VIT_SEED).eval().state_dict()


@pytest.fixture(scope="module")
def ev(state):
    return VitF64(state)


@pytest.fixture(scope="module")
def ctx(state):
    torch.set_num_threads(max(1, min(16, torch.get_num_threads())))
    c = _native.Context.get("cuda:0")
    c.load_vit([v.cuda() for v in state.values()])
    return c


def wide(O, S, sm):
    """enqueue_tc_linear's rule: 128-feature tiles when O % 128 == 0 and they still give every SM a tile."""
    return O % 128 == 0 and (O // 128) * math.ceil(S / 128) >= sm


def frame_counts(sm):
    """{label: n}: the demo / evaluation sizes and, per GEMM width, the last n on 64-feature and the first on 128-feature tiles."""
    out = {"n1": 1, "n2": 2, "n10": 10, "n20": 20}
    for name, O in GEMMS.items():
        first = next(n for n in range(1, 1000) if wide(O, TOKENS * n, sm))
        out[f"{name} last 64-wide"], out[f"{name} first 128-wide"] = first - 1, first
    return out


def check_rows(case, dev, f64, tf, base=None):
    """The bound per row of [rows, 384]; base = the stream before the block (norms of `ref` over the update)."""
    dev = dev.detach().cpu().double()
    ref = f64 - base if base is not None else f64
    err, bound = (dev - f64).norm(dim=-1), 4 * (tf - f64).norm(dim=-1) + 1e-6 * ref.norm(dim=-1)
    ratio = err / bound
    RATIOS[case] = max(RATIOS.get(case, 0.0), ratio.max().item())
    bad = int((err > bound).sum())
    worst = int(ratio.argmax())
    assert bad == 0, f"{case}: {bad} of {len(err)} rows out of bound; row {worst}: error {err[worst]:.3e}, bound {bound[worst]:.3e}"


def check_stages(ctx, ev, case, img, sf, blocks, tf_ev=None, z_ref=None):
    """Stage 0, teacher-forced blocks and z of `img` [n,3,h,w] (CPU) against the evaluator; returns the device z.
    tf_ev: evaluator of the tf32 run (default ev); z_ref: (z f64, z tf32) when precomputed."""
    tf_ev = tf_ev or ev
    n, _, h, w = img.shape
    tokens = tokens_per_scale(h, w, sf)
    dev_img = img.cuda()
    dumps = {}

    def dump(k):
        if k not in dumps:
            dumps[k] = ctx.extract_features(dev_img, sf, debug_stage=k)[1].cpu().double()
        return dumps[k]

    f64 = join_rows([ev.prepare_tokens(p) for p in ev.pyramid(img, sf)])
    tf = join_rows([tf_ev.prepare_tokens(p, "tf32") for p in tf_ev.pyramid(img, sf)])
    check_rows(f"{case} stage 0", dump(0), f64, tf)
    for k in blocks:
        prev = dump(k - 1)
        xs = split_rows(prev, n, tokens)
        f64 = join_rows([ev.block(k, x) for x in xs])
        tf = join_rows([tf_ev.block(k, x, "tf32") for x in xs])
        check_rows(f"{case} blocks", dump(k), f64, tf, base=prev)
        dumps.pop(k - 1)
    z = ctx.extract_features(dev_img, sf)
    z64, ztf = z_ref if z_ref is not None else (ev.features(img, sf), tf_ev.features(img, sf, "tf32"))
    check_rows(f"{case} z", z, z64, ztf)
    return z


# ---- frame counts and tile regimes ----------------------------------------------------------------------------------------
LABELS = ["n1", "n2", "n10", "n20"] + [f"{g} {side}" for g in GEMMS for side in ("last 64-wide", "first 128-wide")]


def test_frame_counts_cover_both_tile_widths_of_every_gemm(ctx):
    sm = ctx.sm_count()
    ns = set(frame_counts(sm).values())
    for name, O in GEMMS.items():
        assert {wide(O, TOKENS * n, sm) for n in ns} == {False, True}, (name, sm, sorted(ns))
    print(f"\n{sm} SMs: frame counts {frame_counts(sm)}")


@pytest.fixture(scope="module")
def frames_ref(ctx, ev):
    """Images (prefixes of one seeded batch) and their float64 / tf32 z, computed once for the largest n."""
    n_max = max(frame_counts(ctx.sm_count()).values())
    img = images_for(n_max, 224, 224, 31)
    return img, ev.features(img, SF), ev.features(img, SF, "tf32")


@pytest.mark.parametrize("label", LABELS)
def test_frame_counts_against_float64(ctx, ev, frames_ref, label):
    counts = frame_counts(ctx.sm_count())
    n = counts[label]
    if label not in ("n1", "n2", "n10", "n20") and any(counts[o] == n for o in LABELS[:LABELS.index(label)]):
        pytest.skip(f"n = {n} is checked by an earlier case")
    img, z64, ztf = frames_ref
    img = img[:n].contiguous()
    z = check_stages(ctx, ev, f"frames n={n}", img, SF, (1, 6, 12), z_ref=(z64[:n], ztf[:n]))
    # the last frame alone (64-feature tiles everywhere) and inside this batch: bit-identical
    assert torch.equal(z[n - 1:], ctx.extract_features(img[n - 1:].cuda(), SF))


def test_training_size_512_images(ctx, ev):
    """A training step's max_images: 512 frames at 224^2 (S = 135 168 rows).  z of 8 sampled frames against float64, and
    bit-identical to those frames run alone."""
    img = images_for(512, 224, 224, 32)
    z = ctx.extract_features(img.cuda(), SF).cpu()
    pick = [0, 1, 100, 255, 256, 384, 510, 511]
    sub = img[pick].contiguous()
    check_rows("train 512 z", z[pick], ev.features(sub, SF), ev.features(sub, SF, "tf32"))
    for i in pick:
        assert torch.equal(z[i:i + 1], ctx.extract_features(img[i:i + 1].cuda(), SF).cpu()), i


# ---- attention lengths ----------------------------------------------------------------------------------------------------
ATT_CASES = [  # (h, w, scale factors): tokens per sequence
    (16, 16, [1]),  # 2
    (16, 112, [1]),  # 8: one full key tile
    (16, 128, [1]),  # 9
    (112, 144, [1]),  # 64: one full key block
    (64, 256, [1]),  # 65
    (112, 288, [1]),  # 127
    (128, 256, [1]),  # 129: second query chunk
    (240, 272, [1]),  # 256: the limit
    (240, 272, [1, 1 / 2, 1 / 3, 1 / 4]),  # 256, 57, 26, 13 in one launch, at the scale limit
    (64, 64, [2]),  # upsampling: 65
]


@pytest.mark.parametrize("h,w,sf", ATT_CASES, ids=[f"{h}x{w}-L{'-'.join(map(str, tokens_per_scale(h, w, sf)))}" for h, w, sf in ATT_CASES])
def test_attention_lengths_against_float64(ctx, ev, h, w, sf):
    img = images_for(3, h, w, 40 + h + w)
    check_stages(ctx, ev, f"attention {h}x{w} L={tokens_per_scale(h, w, sf)}", img, sf, range(1, 13))


# ---- position tables ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("h,w,sf", [(224, 232, [1]), (232, 224, [1]), (224, 239, [1]), (448, 464, [1 / 2]), (224, 224, [1])])
def test_position_table_of_non_square_inputs(ctx, ev, h, w, sf):
    """A 14x14 grid of a non-square image takes the resampled table (scale 14.1 / 14), as the hub model does; 224^2 the stored one."""
    img = images_for(2, h, w, 50)
    check_stages(ctx, ev, f"position table {h}x{w}", img, sf, (1,))


# ---- mean-dominated rows --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [2, 10])
def test_mean_dominated_rows(state, ev, n):
    """pos_embed + 20: every row carries +20 in all channels through every block; each LayerNorm removes it, so z is the
    unshifted network's, while mean * colsum now dominates the folded qkv / fc1 epilogue."""
    shifted = dict(state)
    shifted["pos_embed"] = state["pos_embed"] + 20.0
    sev = VitF64(shifted)
    c = _native.Context(0)
    try:
        c.load_vit([v.cuda() for v in shifted.values()])
        img = images_for(n, 224, 224, 60)
        z64, ztf = ev.features(img, SF), sev.features(img, SF, "tf32")  # z64: the unshifted weights
        zdev = check_stages(c, sev, f"mean-dominated n={n}", img, SF, (1, 6, 12), z_ref=(z64, ztf)).cpu().double()
        zln = sev.features(img, SF, "tf32_ln")
        print(f"\nmean-dominated n={n}: max|z - f64| dev {(zdev - z64).abs().max():.3e}, tf32 folded {(ztf - z64).abs().max():.3e}, "
              f"tf32 explicit LayerNorm {(zln - z64).abs().max():.3e}; max|dev - tf32 explicit LayerNorm| {(zdev - zln).abs().max():.3e}")
    finally:
        c.lib.pdb_destroy(c.handle)


# ---- swap-AB tiles --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,h,w", [(1, 64, 64), (5, 16, 16)])
def test_swap_ab_tiles_with_the_vit_epilogues(ctx, ev, n, h, w):
    img = images_for(n, h, w, 70)
    ctx.set_tc_swap(True)
    try:
        check_stages(ctx, ev, f"swap-AB {n}x{h}x{w}", img, [1], range(1, 13))
    finally:
        ctx.set_tc_swap(False)


# ---- refusals -------------------------------------------------------------------------------------------------------------
def test_refusals_leave_the_context_usable(ctx):
    img = images_for(2, 224, 224, 80).cuda()
    before = ctx.extract_features(img, SF)
    limit, invalid = rf"failed \({_native.PDB_ERR_LIMIT}\)", rf"failed \({_native.PDB_ERR_INVALID}\)"
    with pytest.raises(_native.NativeError, match=limit):
        ctx.extract_features(torch.rand(1, 3, 256, 256, device="cuda"), [1])  # 257 tokens
    with pytest.raises(_native.NativeError, match=limit):
        ctx.extract_features(img, [1, 1 / 2, 1 / 3, 1 / 4, 1 / 5])
    for bad in (float("nan"), 0.0):
        with pytest.raises(_native.NativeError, match=invalid):
            ctx.extract_features(img, [1, bad])
    many = torch.zeros(65536, 3, 16, 16, device="cuda")  # image index on gridDim.y: refused on the host
    launches = ctx.launch_count
    with pytest.raises(_native.NativeError, match=limit):
        ctx.extract_features(many, [1])
    assert ctx.launch_count == launches
    del many
    assert torch.equal(ctx.extract_features(img, SF), before)
