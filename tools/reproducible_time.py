#!/usr/bin/env python
"""Cost of reproducible sampling (torch.use_deterministic_algorithms -> pdb_set_reproducible): one full p_sample_loop (T = 100)
per run in the default and the reproducible mode, alternating, at the bench.py workloads it changes:

    cfg3        1 x 20 frames, GGS on (380 ordered pairs x 2048 matches, resident slices)
    cfg4_share  8 x 20 frames, GGS on (config 4's share of one GPU; tensor-core denoiser engine)
    cfg5_stream 1 x 80 frames, GGS on (6320 ordered pairs x 4096 matches: 25.9 M, streamed through the bulk-async ring)
    unguided    8 x 20 frames, GGS off (tensor-core denoiser engine alone)

Medians (and min / max) of --runs runs per mode in ms per loop, from CUDA events around the loop.  Also dumps the cfg3 pose twice
per mode and says whether the two dumps have the same bits: the A/B check between builds that reproducible mode makes possible.

    python tools/reproducible_time.py [--runs 7] [--workloads cfg3,cfg4_share,cfg5_stream,unguided] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import posediffusion_b200 as pdb  # noqa: E402
from posediffusion_b200 import synthetic as syn  # noqa: E402

WORKLOADS = {  # batch, frames, matches per ordered pair (0: GGS off)
    "cfg3": (1, 20, 2048),
    "cfg4_share": (8, 20, 2048),
    "cfg5_stream": (1, 80, 4096),
    "unguided": (8, 20, 0),
}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="directory for the JSON record")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    den = pdb.Denoiser(TRANSFORMER=dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1,
                                        batch_first=True, norm_first=True))
    den.load_state_dict(syn.random_denoiser_state(args.seed), strict=True)
    den = den.to(dev)
    ctx = den.native_context()
    cfg = syn.default_ggs_cfg()
    cfg["verbose"] = False
    record = {"gpu": gpu_info(), "runs": args.runs, "workloads": {}}
    print(f"# {record['gpu']}")
    before = torch.are_deterministic_algorithms_enabled()
    try:
        for name in args.workloads.split(","):
            B, N, per_pair = WORKLOADS[name]
            z = torch.cat([syn.random_features(1, N, args.seed + b) for b in range(B)]).to(dev)
            draws = torch.cat([syn.predraw_noise(1, N, seed=args.seed + b) for b in range(B)], dim=1).contiguous().to(dev)
            problems = [ctx.pack_matches(syn.uniform_matches(N, per_pair, seed=args.seed + b)) for b in range(B)] if per_pair else None
            start = cfg["start_step"] if per_pair else 0
            stream = name == "cfg5_stream"
            if stream:  # force the ring even where the slices would fit in shared memory
                os.environ["PDB_GGS_FORCE_STREAM"] = "1"

            def loop():
                return ctx.sample_loop(z, draws, problems, cfg if per_pair else None, start, want_trail=False, want_stats=False)[0]

            times = {"default": [], "reproducible": []}
            dumps = {"default": [], "reproducible": []}
            for mode in ("default", "reproducible"):  # warm-up: modules, graphs and workspaces of both modes
                torch.use_deterministic_algorithms(mode == "reproducible")
                loop()
            torch.cuda.synchronize()
            for r in range(args.runs):
                for mode in (("default", "reproducible") if r % 2 == 0 else ("reproducible", "default")):
                    torch.use_deterministic_algorithms(mode == "reproducible")
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    pose = loop()
                    b.record()
                    b.synchronize()
                    times[mode].append(a.elapsed_time(b))
                    if len(dumps[mode]) < 2:
                        dumps[mode].append(pose.cpu().numpy().tobytes())
            if stream:
                del os.environ["PDB_GGS_FORCE_STREAM"]
            res = {m: {"median_ms": float(np.median(t)), "min_ms": float(np.min(t)), "max_ms": float(np.max(t))} for m, t in times.items()}
            res["cost"] = res["reproducible"]["median_ms"] / res["default"]["median_ms"] - 1.0
            res["same_bits_twice"] = {m: d[0] == d[1] for m, d in dumps.items()}
            record["workloads"][name] = res
            print(f"{name:12s} default {res['default']['median_ms']:8.2f} ms  reproducible {res['reproducible']['median_ms']:8.2f} ms  "
                  f"cost {100 * res['cost']:+6.1f} %  same bits twice: default {res['same_bits_twice']['default']}, "
                  f"reproducible {res['same_bits_twice']['reproducible']}")
    finally:
        torch.use_deterministic_algorithms(before)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "reproducible_time.json"), "w") as f:
            json.dump(record, f, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
