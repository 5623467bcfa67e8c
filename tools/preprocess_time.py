"""Time image preprocessing: the reference's CPU path against pdb_images_preprocess_host.  Prints one JSON line.

    python tools/preprocess_time.py [--frames 20] [--height 1066] [--width 1896] [--reps 10]

Workload: seeded frames of the sample sequence's size (1066 x 1896), encoded as JPEG (quality 95) for the decode timings and held
decoded in host memory for the preprocessing timings.  Every time is host wall clock; the native call synchronises its stream
before returning.  Needs a CUDA device (no fallback).
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import tempfile
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import preprocess_oracle  # noqa: E402
from oracle.make_golden_preprocess import frames_for  # noqa: E402
from posediffusion_b200 import _native  # noqa: E402
from posediffusion_b200.load_img_folder import center_crop_geometry, decode_image  # noqa: E402


def touched_rows(side: int, size: int) -> int:
    """Crop rows the bilinear resize reads (the index arithmetic of csrc/preprocess.cuh, restated)."""
    scale = np.float32(side) / np.float32(size)
    src = np.maximum(np.float64(scale) * (np.arange(size, dtype=np.float64) + 0.5) - 0.5, 0.0).astype(np.float32)
    i0 = np.minimum(src.astype(np.int64), side - 1)
    i1 = i0 + (i0 < side - 1)
    return len(np.union1d(i0, i1))


def timed(fn, reps):
    out, times = None, []
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return out, times


def stats(times):
    return {"median_ms": round(float(np.median(times)), 3), "min_ms": round(min(times), 3), "max_ms": round(max(times), 3), "reps": len(times)}


def gpu_power_limit() -> str:
    try:
        res = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                             text=True, timeout=30)
        return res.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--height", type=int, default=1066)
    ap.add_argument("--width", type=int, default=1896)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    nproc = os.cpu_count() or 1
    torch.set_num_threads(nproc)
    ctx = _native.Context.get("cuda:0")
    frames = frames_for([(args.height, args.width)] * args.frames, 2024)
    with tempfile.TemporaryDirectory() as tmp:
        paths = []
        for i, f in enumerate(frames):
            paths.append(os.path.join(tmp, f"{i:03d}.jpg"))
            Image.fromarray(f).save(paths[-1], quality=95)
        decode_image(paths[0])  # warm the codec
        _, serial = timed(lambda: [decode_image(p) for p in paths], 3)
        with ThreadPoolExecutor(max_workers=min(len(paths), nproc)) as pool:
            _, threaded = timed(lambda: list(pool.map(decode_image, paths)), 3)
    crops, _ = center_crop_geometry([f.shape[:2] for f in frames], args.size)
    preprocess_oracle.preprocess(frames[:2], args.size)
    ref, cpu_times = timed(lambda: preprocess_oracle.preprocess(frames, args.size)[0], 3)
    for _ in range(3):  # warm-up: staging buffers, module load
        ctx.preprocess_images(frames, crops, args.size)
    got, gpu_times = timed(lambda: ctx.preprocess_images(frames, crops, args.size), max(args.reps, 5))
    side = int(crops[0][2])
    uploaded = sum(touched_rows(int(c[2]), args.size) * 3 * int(c[2]) + 8 * args.size for c in crops)
    print(json.dumps({
        "gpu": torch.cuda.get_device_name(0), "power_limit": gpu_power_limit(), "nproc": nproc,
        "workload": f"{args.frames} frames {args.height}x{args.width} -> {args.size}^2",
        "pil_decode_serial": stats(serial), "pil_decode_threaded": stats(threaded),
        "cpu_convert_crop_interpolate": stats(cpu_times), "torch_threads": torch.get_num_threads(),
        "pdb_images_preprocess_host": stats(gpu_times),
        "touched_rows_per_frame": touched_rows(side, args.size), "crop_side": side,
        "bytes_uploaded": uploaded, "bytes_full_frames": sum(f.nbytes for f in frames),
        "max_abs_diff_vs_cpu": float((got.cpu() - ref).abs().max().item()),
    }))


if __name__ == "__main__":
    main()
