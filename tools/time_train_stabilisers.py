"""Per-step time of `train_auto`'s graph-replayed epoch with gradient-norm clipping and / or an EMA of the weights,
against the same epoch without either, on the same seeded split.

    python tools/time_train_stabilisers.py [--cases 20] [--frames 51] [--reps 5] \
        [--out profiles/train_stabilisers_h100.json]

For each workload (cavity 64x64 in fp32 and bf16 storage, tube 66x65) and batch size (8, 64, 256) it times one
single-step epoch (_StepGraphs, no evaluation) of four step graphs that differ only in the optimizer:
  * "none": FusedAdam(lr) -- the step graph train_auto runs by default;
  * "clip": FusedAdam(lr, max_grad_norm=1.0) -- plus the global-norm launch and the clipping Adam;
  * "ema": FusedAdam(lr, ema_decay=0.9999) -- the Adam launch also updates the EMA;
  * "both": both options.
Each is a host clock around one epoch (uploads, one graph replay per step, the log copied back) that ends in a device
synchronise; the four alternate, and the median of `--reps` repetitions is reported per step with the minimum and
maximum.  The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cfdbench_b200 import DeviceFrames, FusedAdam, synth  # noqa: E402
from cfdbench_b200.train import _StepGraphs, epoch_permutation  # noqa: E402
from test_gpu_eval_auto import _model  # noqa: E402
from test_gpu_train_rollout import _ChainSplit  # noqa: E402
from time_train_rollout_epoch import _card  # noqa: E402

MODES = {"none": {}, "clip": dict(max_grad_norm=1.0), "ema": dict(ema_decay=0.9999),
         "both": dict(max_grad_norm=1.0, ema_decay=0.9999)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=20)
    ap.add_argument("--frames", type=int, default=51, help="frames per case (samples per case = frames - 1)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", default="8,64,256")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "train_stabilisers_h100.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool times the GPU"
    card = _card()
    print("card:", card)
    rows = []
    for problem, act in (("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32")):
        ds = _ChainSplit([args.frames] * args.cases, problem, s=1, seed=0)
        frames = DeviceFrames(ds, device="cuda")
        for b in (int(x) for x in args.batches.split(",")):
            impls, state = {}, {}
            for name, opts in MODES.items():
                m = _model(problem, act, seed=1)
                opt = FusedAdam(m.parameters(), lr=1e-3, **opts)
                graphs = _StepGraphs(m, frames, b, opt)
                state[name] = dict(graphs=graphs, gen=torch.Generator().manual_seed(0), step=0, model=m)

                def run(s=state[name]):
                    perm = epoch_permutation(frames.n, b, s["gen"])
                    s["graphs"].epoch(perm, 1e-3, s["step"] + 1)
                    s["step"] += s["graphs"].steps
                    torch.cuda.synchronize()
                impls[name] = run
            times = {k: [] for k in impls}
            for fn in impls.values():   # warm-up epoch of every mode
                fn()
            for _ in range(args.reps):
                for k, fn in impls.items():
                    t0 = time.perf_counter()
                    fn()
                    times[k].append(time.perf_counter() - t0)
            steps = state["none"]["graphs"].steps
            med = {k: statistics.median(v) for k, v in times.items()}
            row = dict(problem=problem, grid=list(synth.grid(problem)), act_dtype=act, batch=b, steps=steps,
                       epoch_s=times, spread_step_ms={k: [1e3 * min(v) / steps, 1e3 * max(v) / steps]
                                                      for k, v in times.items()},
                       median_step_ms={k: 1e3 * v / steps for k, v in med.items()},
                       overhead_vs_none_pct={k: 100.0 * (med[k] / med["none"] - 1.0) for k in med if k != "none"})
            rows.append(row)
            print(json.dumps({k: row[k] for k in ("problem", "act_dtype", "batch", "median_step_ms",
                                                  "overhead_vs_none_pct")}), flush=True)
            del impls, state
            torch.cuda.empty_cache()
    rec = dict(tool="tools/time_train_stabilisers.py", card=card, torch=torch.__version__, reps=args.reps,
               split=dict(cases=args.cases, frames_per_case=args.frames),
               modes={k: dict(v) for k, v in MODES.items()},
               timing="host clock around one single-step epoch ending in torch.cuda.synchronize(), divided by the "
                      "epoch's steps; median of alternating reps, spread = [min, max]",
               rows=rows)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
