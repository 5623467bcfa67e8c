"""Image preprocessing (load_and_preprocess_images) without a GPU: the crop geometry helper, file listing and error behaviour of
posediffusion_b200.load_img_folder, the CPU oracle, and csrc/preprocess.cuh compiled for the host (tests/host/preprocess_host.cu:
the staging planner and the kernel body) against the fixtures the reference's own function produced."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import load_golden
from oracle import preprocess_oracle
from oracle.make_golden_preprocess import CASES, frames_for, images_for
from posediffusion_b200 import _native
from posediffusion_b200.load_img_folder import center_crop_geometry, decode_image, list_images, load_and_preprocess_images

TOL = 3e-7  # values in [0, 1]; 1 ulp at 1.0 is 1.19e-7


@pytest.fixture(scope="module")
def host():
    import __graft_entry__ as entry

    lib = C.CDLL(entry.build_preprocess_harness())
    lib.pre_host_plan_misses.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.pre_host_tap.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    lib.pre_host_run.argtypes = [C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def decoded(tmp_path_factory):
    folder = tmp_path_factory.mktemp("png")
    return {case: [decode_image(p) for p in images_for(case, str(folder))] for case in CASES}


def host_run(lib, frames, crops, size):
    keep = [np.ascontiguousarray(f) for f in frames]
    ptrs = (C.c_void_p * len(keep))(*[f.ctypes.data for f in keep])
    hw = np.asarray([f.shape[:2] for f in keep], dtype=np.int32)
    crops = np.ascontiguousarray(crops, dtype=np.int32)
    out = np.empty((len(keep), 3, size, size), dtype=np.float32)
    assert lib.pre_host_run(len(keep), ptrs, hw.ctypes.data, crops.ctypes.data, size, out.ctypes.data) == 0
    return out


@pytest.mark.parametrize("case", list(CASES))
def test_geometry_matches_reference_exactly(golden, case):
    size, specs, _ = CASES[case]
    g = golden("preprocess.npz")
    crops, info = center_crop_geometry([(h, w) for h, w, _ in specs], size)
    assert info["bboxes_xyxy"].dtype == np.int64 and np.array_equal(info["bboxes_xyxy"], g[f"{case}_bboxes"])
    assert info["resized_scales"].dtype == np.float64 and np.array_equal(info["resized_scales"], g[f"{case}_scales"])
    assert info["size"] == tuple(int(v) for v in g[f"{case}_size"])  # the LAST frame's crop side
    assert np.array_equal(crops[:, 2], g[f"{case}_bboxes"][:, 2] - g[f"{case}_bboxes"][:, 0])


@pytest.mark.parametrize("case", list(CASES))
def test_oracle_is_bit_exact_with_reference(golden, decoded, case):
    threads = torch.get_num_threads()
    torch.set_num_threads(1)  # the fixture's setting (ATen's resize loop depends on it; see oracle/make_golden_preprocess.py)
    try:
        images, bboxes, scales = preprocess_oracle.preprocess(decoded[case], CASES[case][0])
    finally:
        torch.set_num_threads(threads)
    g = golden("preprocess.npz")
    assert np.array_equal(images.numpy(), g[f"{case}_images"])
    assert np.array_equal(bboxes, g[f"{case}_bboxes"]) and np.array_equal(scales, g[f"{case}_scales"])


@pytest.mark.parametrize("case", list(CASES))
def test_kernel_body_on_host_matches_reference(host, golden, decoded, case):
    size = CASES[case][0]
    crops, _ = center_crop_geometry([f.shape[:2] for f in decoded[case]], size)
    out = host_run(host, decoded[case], crops, size)
    ref = golden("preprocess.npz")[f"{case}_images"]
    assert np.abs(out - ref).max() <= TOL, np.abs(out - ref).max()
    if case == "identity":
        assert np.array_equal(out, ref)


@pytest.mark.parametrize("side,size", [(1066, 224), (1896, 224), (173, 224), (40, 224), (500, 224), (224, 224), (75, 64),
                                       (2, 64), (2, 1), (64, 2), (300, 224), (449, 224), (448, 224)])
def test_plan_stages_every_row_the_kernel_reads(host, side, size):
    rows = np.zeros(side, dtype=np.int32)
    count = C.c_int()
    assert host.pre_host_plan_misses(side, size, rows.ctypes.data, C.byref(count)) == 0
    staged = rows[: count.value]
    assert np.all(np.diff(staged) > 0) and count.value <= min(side, 2 * size)
    taps = np.zeros(2, dtype=np.int32)
    w = np.zeros(2, dtype=np.float32)
    read = set()
    for y in range(size):
        host.pre_host_tap(y, side, size, taps.ctypes.data, w.ctypes.data)
        read.update(int(t) for t in taps)
    assert read == set(staged.tolist())  # staged rows are exactly the rows read


def test_full_size_frame_against_oracle(host):
    """One 1066x1896 frame (the sample sequence's portrait size, transposed here) through the host kernel body vs ATen."""
    frame = frames_for([(1066, 1896)], 41)[0]
    crops, _ = center_crop_geometry([frame.shape[:2]], 224)
    out = host_run(host, [frame], crops, 224)
    ref = preprocess_oracle.preprocess([frame], 224)[0].numpy()
    assert np.abs(out - ref).max() <= TOL, np.abs(out - ref).max()


def test_listing_filters_extensions_and_sorts_in_place(tmp_path):
    for name in ("b.PNG", "a.jpeg", "c.JpG", "notes.txt", "d.png.bak", "e.gif"):
        (tmp_path / name).write_bytes(b"")
    assert sorted(list_images(str(tmp_path))) == [str(tmp_path / n) for n in ("a.jpeg", "b.PNG", "c.JpG")]
    paths = ["z.png", "a.png", "m.jpg"]
    with pytest.raises(NotImplementedError):  # raised after the in-place sort, like the reference's ordering of side effects
        load_and_preprocess_images(image_paths=paths, mode="bicubic")
    assert paths == ["a.png", "m.jpg", "z.png"]


def test_error_paths_without_device(tmp_path):
    with pytest.raises(ValueError):
        load_and_preprocess_images(image_paths=[])
    with pytest.raises(ValueError):
        load_and_preprocess_images(folder_path=str(tmp_path))  # no image files
    with pytest.raises(ValueError):
        center_crop_geometry([], 224)
    from PIL import Image

    Image.fromarray(np.zeros((1, 7, 3), dtype=np.uint8)).save(tmp_path / "thin.png")
    with pytest.raises(ValueError, match="squashed image"):
        load_and_preprocess_images(folder_path=str(tmp_path))
    with pytest.raises(ValueError, match="squashed image"):
        center_crop_geometry([(40, 1)], 224)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-fallback error of a CPU-only machine")
def test_cpu_only_raises_native_error(tmp_path):
    Image = pytest.importorskip("PIL.Image")
    Image.fromarray(frames_for([(20, 30)], 3)[0]).save(tmp_path / "f.png")
    with pytest.raises(_native.NativeError):
        load_and_preprocess_images(folder_path=str(tmp_path), image_size=16)
