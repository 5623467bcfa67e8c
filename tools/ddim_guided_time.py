"""Loop time of guided DDIM jumps: the guided tail in g' = 10, 5, 2 and 1 denoiser evaluations after a k = 10 DDIM prefix.

    python tools/ddim_guided_time.py [--loops 7] [--warmup 3] [--out DIR]

Two workloads with GGS on (start_step g = 10, 700 inner iterations per guided step, iteration counts not rescaled by the stride),
each over geometry-consistent scenes of 20 frames x 380 ordered pairs x 2048 matches (778 240 per sequence):
  * cfg3: one sequence (the fp32 persistent denoiser engine);
  * the 8 x 20 share of cfg4: eight sequences on one GPU (the tensor-core engine).
Each variant runs what `GaussianDiffusion.ddim_sample(sampling_timesteps = 10 + g', eta = 0, guided_steps = g')` runs, through the
same context call with a pre-made x_T.  Loops are timed with CUDA events on the sampling stream, calls alternating between the
variants so that clock and neighbour drift hit them alike; the median of `--loops` loops per variant after `--warmup` untimed ones.
The denoiser and GGS device milliseconds per loop come from pdb_profile_read.  As a guidance proxy the table also gives the
Sampson error GGS logs in the last phase of the last guided jump (mean over sequences, from the last timed loop).  The denoiser's
weights are random, so this is not pose accuracy.  Prints the GPU's name, power limit and SM clocks first; writes
ddim_guided_time.json under --out when given.
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
from posediffusion_b200 import _native  # noqa: E402
from posediffusion_b200 import synthetic as syn  # noqa: E402

TRANSFORMER = dict(d_model=512, nhead=4, dim_feedforward=1024, num_encoder_layers=8, dropout=0.1, batch_first=True, norm_first=True)
K = 10
GUIDED = (10, 5, 2, 1)


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
    g = cfg["start_step"]
    rows = []
    for name, B in (("cfg3 (B1 N20, 778 240 matches)", 1), ("8 x 20 share of cfg4 (778 240 matches each)", 8)):
        N = 20
        z = syn.random_features(B, N, 1).to(dev)
        x_T = torch.randn(1, B, N, 9, generator=torch.Generator().manual_seed(1)).to(dev)
        problems = [ctx.pack_matches(syn.scene_matches(N, 2048, seed=1 + b, ordered=True)[0]) for b in range(B)]
        variants = [(gs, lambda gs=gs: ctx.sample_loop_ddim(z, x_T, K + gs, 0.0, problems, cfg, g, want_trail=False,
                                                            guided_steps=gs)) for gs in GUIDED]
        for _ in range(args.warmup):
            for _, fn in variants:
                fn()
        torch.cuda.synchronize()
        ctx.profile(True)
        ctx.profile_read()
        res = {gs: {"ms": [], "den": [], "ggs": [], "sampson": None} for gs, _ in variants}
        for _ in range(args.loops):
            for gs, fn in variants:
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                _, _, stats = fn()
                b.record()
                torch.cuda.synchronize()
                ggs_ms, _, den_ms, _ = ctx.profile_read()
                res[gs]["ms"].append(a.elapsed_time(b))
                res[gs]["den"].append(den_ms)
                res[gs]["ggs"].append(ggs_ms)
                last = _native.stats_to_numpy(stats).reshape(gs, B)[-1]
                res[gs]["sampson"] = float(last["sampson"][:, -1].mean())
        ctx.profile(False)
        for gs, _ in variants:
            r = res[gs]
            rows.append({"workload": name, "guided_steps": gs, "evaluations": K + gs, "loop_ms": statistics.median(r["ms"]),
                         "loop_ms_min": min(r["ms"]), "loop_ms_max": max(r["ms"]), "denoiser_ms": statistics.median(r["den"]),
                         "ggs_ms": statistics.median(r["ggs"]), "last_jump_sampson": r["sampson"]})
    print(f"{'workload':44s} {'g_':>3s} {'evals':>5s} {'loop ms':>9s} {'(min..max)':>17s} {'denoiser ms':>11s} {'GGS ms':>8s} "
          f"{'last Sampson':>12s}")
    for r in rows:
        print(f"{r['workload']:44s} {r['guided_steps']:3d} {r['evaluations']:5d} {r['loop_ms']:9.3f} "
              f"({r['loop_ms_min']:7.3f}..{r['loop_ms_max']:7.3f}) {r['denoiser_ms']:11.3f} {r['ggs_ms']:8.3f} "
              f"{r['last_jump_sampson']:12.5f}")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ddim_guided_time.json"), "w") as fh:
            json.dump({"gpu": card(), "loops": args.loops, "rows": rows}, fh, indent=1)
    return 0


if __name__ == "__main__":
    sys.exit(main())
