"""Loop time of fewer-step sampling: `sample()`'s DDPM loop against DDIM prefixes of k = 10, 20 and 45 steps.

    python tools/ddim_time.py [--loops 7] [--warmup 3] [--out DIR]

Three workloads, each loop timed with CUDA events on the sampling stream, calls alternating between the variants so that clock
and neighbour drift hit them alike; the median of `--loops` loops per variant after `--warmup` untimed ones:
  * B1 N20, GGS off (the fp32 persistent engine; bench.py cfg2);
  * cfg3: B1 N20, GGS on with start_step 10 over 380 ordered pairs x 2048 matches (778 240), 700 inner iterations per guided step;
  * 8 x 20 = 160 tokens, GGS off (the tensor-core engine).
The variants run what `GaussianDiffusion.sample` and `.ddim_sample(sampling_timesteps = k + g, eta = 0)` run, through the same
context calls with pre-made draws (no trajectory copy-out); g = 10 guided steps on cfg3, else 0.  The denoiser and GGS device
milliseconds per loop come from pdb_profile_read.  Prints the GPU's name, power limit and SM clock first, then one table; writes
ddim_time.json under --out when given.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402

import posediffusion_b200 as pdb  # noqa: E402
from posediffusion_b200 import synthetic as syn  # noqa: E402

TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
KS = (10, 20, 45)


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as exc:
        return f"nvidia-smi unavailable ({exc})"


def main() -> int:
    ap = argparse.ArgumentParser()
    ap.add_argument("--loops", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures on the GPU only")
    dev = torch.device("cuda:0")
    print(f"GPU: {card()}  (name, power limit, SM clock now, max SM clock)")
    den = pdb.Denoiser(TRANSFORMER=TRANSFORMER)
    den.load_state_dict(syn.random_denoiser_state(0), strict=True)
    den = den.to(dev)
    ctx = den.native_context()
    cfg = syn.default_ggs_cfg()
    cfg["verbose"] = False
    workloads = [("B1 N20, GGS off", 1, 20, 0), ("cfg3 (B1 N20, 778 240 matches, GGS on)", 1, 20, 2048),
                 ("8 x 20, GGS off (tensor cores)", 8, 20, 0)]
    rows = []
    for name, B, N, per_pair in workloads:
        z = syn.random_features(B, N, 1).to(dev)
        draws = syn.predraw_noise(B, N, seed=1).to(dev)
        x_T = draws[:1].contiguous()
        problems = [ctx.pack_matches(syn.uniform_matches(N, per_pair, seed=1 + b)) for b in range(B)] if per_pair else None
        g = cfg["start_step"] if per_pair else 0
        variants = [("sample() DDPM", lambda: ctx.sample_loop(z, draws, problems, cfg if problems else None, g, want_trail=False,
                                                                want_stats=False))]
        for k in KS:
            variants.append((f"ddim k={k}", lambda k=k: ctx.sample_loop_ddim(z, x_T, k + g, 0.0, problems, cfg if problems else None, g,
                                                                            want_trail=False, want_stats=False)))
        for _ in range(args.warmup):
            for _, fn in variants:
                fn()
        torch.cuda.synchronize()
        ctx.profile(True)
        ctx.profile_read()
        res = {v: {"ms": [], "den": [], "ggs": []} for v, _ in variants}
        for _ in range(args.loops):
            for v, fn in variants:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                fn()
                b.record()
                torch.cuda.synchronize()
                ggs_ms, _, den_ms, _ = ctx.profile_read()
                res[v]["ms"].append(a.elapsed_time(b))
                res[v]["den"].append(den_ms)
                res[v]["ggs"].append(ggs_ms)
        ctx.profile(False)
        for v, _ in variants:
            r = res[v]
            rows.append({"workload": name, "variant": v, "evaluations": (100 if v.startswith("sample") else int(v.split("=")[1]) + g),
                         "loop_ms": statistics.median(r["ms"]), "loop_ms_min": min(r["ms"]), "loop_ms_max": max(r["ms"]),
                         "denoiser_ms": statistics.median(r["den"]), "ggs_ms": statistics.median(r["ggs"])})
    print(f"{'workload':42s} {'variant':14s} {'evals':>5s} {'loop ms':>9s} {'(min..max)':>17s} {'denoiser ms':>11s} {'GGS ms':>8s}")
    for r in rows:
        print(f"{r['workload']:42s} {r['variant']:14s} {r['evaluations']:5d} {r['loop_ms']:9.3f} "
              f"({r['loop_ms_min']:7.3f}..{r['loop_ms_max']:7.3f}) {r['denoiser_ms']:11.3f} {r['ggs_ms']:8.3f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ddim_time.json"), "w") as fh:
            json.dump({"gpu": card(), "loops": args.loops, "rows": rows}, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
