"""Image preprocessing on the GPU (pdb_images_preprocess_host, csrc/api_pre.cu + csrc/preprocess.cuh) against the fixtures the
reference's load_and_preprocess_images produced and, at full size, against the CPU oracle (ATen's resize).  Values lie in [0, 1];
the tolerance is 3e-7 absolute (1 ulp at 1.0 is 1.19e-7; ATen's own scalar and vectorised loops differ by up to 1.8e-7)."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import preprocess_oracle
from oracle.make_golden_preprocess import CASES, frames_for, images_for
from posediffusion_b200 import _native
from posediffusion_b200.load_img_folder import center_crop_geometry, load_and_preprocess_images

pytestmark = pytest.mark.gpu
TOL = 3e-7


@pytest.fixture(scope="module")
def ctx():
    return _native.Context.get("cuda:0")


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    d = tmp_path_factory.mktemp("png")
    return {case: images_for(case, str(d)) for case in CASES}


@pytest.mark.parametrize("case", list(CASES))
def test_golden_cases(golden, folder, case):
    size = CASES[case][0]
    images, info = load_and_preprocess_images(image_size=size, image_paths=list(folder[case]))
    g = golden("preprocess.npz")
    assert images.is_cuda and images.dtype == torch.float32 and images.shape == g[f"{case}_images"].shape
    err = np.abs(images.cpu().numpy() - g[f"{case}_images"]).max()
    assert err <= TOL, err
    if case == "identity":
        assert np.array_equal(images.cpu().numpy(), g[f"{case}_images"])
    assert np.array_equal(info["bboxes_xyxy"], g[f"{case}_bboxes"]) and np.array_equal(info["resized_scales"], g[f"{case}_scales"])
    assert info["size"] == tuple(int(v) for v in g[f"{case}_size"])


@pytest.mark.parametrize("shape", [(1066, 1896), (1896, 1066)])
def test_full_size_sequence_against_oracle(ctx, shape):
    frames = frames_for([shape] * 20, 1000 + shape[0])
    crops, _ = center_crop_geometry([f.shape[:2] for f in frames], 224)
    got = ctx.preprocess_images(frames, crops, 224).cpu()
    ref = preprocess_oracle.preprocess(frames, 224)[0]
    err = (got - ref).abs().max().item()
    assert err <= TOL, err


def test_frame_alone_equals_frame_in_mixed_batch(ctx):
    shapes = [(75, 133), (1066, 1896), (57, 40), (224, 300), (1896, 1066)]
    frames = frames_for(shapes, 77)
    crops, _ = center_crop_geometry(shapes, 224)
    batch = ctx.preprocess_images(frames, crops, 224)
    for i in range(len(frames)):
        alone = ctx.preprocess_images(frames[i:i + 1], crops[i:i + 1], 224)
        assert torch.equal(alone[0], batch[i]), i


def test_abi_error_paths(ctx):
    lib = ctx.lib
    frame = frames_for([(40, 50)], 1)[0]
    ptrs = (C.c_void_p * 1)(frame.ctypes.data)
    hw = np.array([[40, 50]], dtype=np.int32)
    out = torch.empty(1, 3, 16, 16, device=ctx.device)
    st = _native._stream_ptr(ctx.device)

    def call(n=1, p=ptrs, h=hw.ctypes.data, crop=(0, 5, 40), size=16, o=out.data_ptr()):
        c = np.array([crop], dtype=np.int32)
        return lib.pdb_images_preprocess_host(ctx.handle, n, p, h, c.ctypes.data, size, o, st)

    assert call() == _native.PDB_OK
    for kwargs in (dict(n=0), dict(n=-1), dict(size=0), dict(size=-3), dict(p=None), dict(h=None), dict(o=None),
                   dict(p=(C.c_void_p * 1)(None)), dict(crop=(1, 5, 40)), dict(crop=(0, 11, 40)), dict(crop=(-1, 0, 10)),
                   dict(crop=(0, 0, 1)), dict(crop=(0, 0, 0))):
        assert call(**kwargs) == _native.PDB_ERR_INVALID, kwargs
    assert lib.pdb_images_preprocess_host(None, 1, ptrs, hw.ctypes.data, hw.ctypes.data, 16, out.data_ptr(), st) == _native.PDB_ERR_INVALID
    with pytest.raises(_native.NativeError, match="outside"):
        ctx.preprocess_images([frame], [(0, 20, 40)], 16)
    with pytest.raises(_native.NativeError, match="expected"):
        ctx.preprocess_images([frame[..., 0]], [(0, 5, 40)], 16)
    with pytest.raises(_native.NativeError, match="crops"):
        ctx.preprocess_images([frame, frame], [(0, 5, 40)], 16)


def test_python_error_paths(folder):
    paths = list(folder["portrait"])
    with pytest.raises(NotImplementedError):
        load_and_preprocess_images(image_paths=paths, mode="nearest")
    with pytest.raises(ValueError):
        load_and_preprocess_images(image_paths=[])


def test_features_of_native_images_match_oracle_images(folder):
    """End to end: MultiScaleImageFeatureExtractor on natively preprocessed images vs on oracle-preprocessed ones (final-feature
    tolerance of test_gpu_features.py)."""
    import posediffusion_b200 as pdb
    from oracle.dino_vit import DinoViTSmall16, randomize
    from oracle.make_golden_features import VIT_SEED

    frames = frames_for([(1066, 1896), (1896, 1066), (300, 401)], 5)
    crops, _ = center_crop_geometry([f.shape[:2] for f in frames], 224)
    ext = pdb.MultiScaleImageFeatureExtractor(freeze=True)
    ext._net.load_state_dict(randomize(DinoViTSmall16(), VIT_SEED).state_dict(), strict=True)
    ext = ext.cuda()
    native = _native.Context.get("cuda:0").preprocess_images(frames, crops, 224)
    ref = preprocess_oracle.preprocess(frames, 224)[0].cuda()
    z_native, z_ref = ext(native), ext(ref)
    assert (z_native - z_ref).abs().max().item() <= 2e-2


def test_colmap_packing_with_native_image_info(ctx, folder):
    """pack_colmap_matches with the image_info of load_and_preprocess_images == with the oracle's."""
    from oracle.make_golden import synthetic_colmap_tables
    from posediffusion_b200 import synthetic as syn
    from posediffusion_b200.load_img_folder import decode_image
    from posediffusion_b200.match_extraction import pack_colmap_matches

    paths = list(folder["mixed"]) + list(folder["landscape_odd"])
    _, info = load_and_preprocess_images(image_size=224, image_paths=paths)
    _, bboxes, scales = preprocess_oracle.preprocess([decode_image(p) for p in sorted(paths)], 224)
    matches, keypoints, _ = synthetic_colmap_tables()
    img_shape = (5, 3, 224, 224)
    pm_native = pack_colmap_matches(ctx, matches, keypoints, info, img_shape)
    pm_oracle = pack_colmap_matches(ctx, matches, keypoints, {"bboxes_xyxy": bboxes, "resized_scales": scales}, img_shape)
    assert (pm_native.m_total, pm_native.segments, pm_native.rounds) == (pm_oracle.m_total, pm_oracle.segments, pm_oracle.rounds)
    pose = torch.from_numpy(syn.scene_matches(5, 4, seed=1)[2]).cuda()
    g1, s1, F1, G1 = ctx.sampson_eval(pm_native, pose, sampson_max=1e9, dump=True)
    g2, s2, F2, G2 = ctx.sampson_eval(pm_oracle, pose, sampson_max=1e9, dump=True)
    assert s1[1].item() == s2[1].item() and torch.equal(F1, F2)
    assert (G1 - G2).abs().max().item() <= 1e-4 * G1.abs().max().item()  # same matches; summation order of the reduction may differ
