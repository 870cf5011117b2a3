"""Epoch time of `train_auto`'s graph-replayed steps against the eager loop a user writes today, on the same seeded split.

    python tools/time_train_epoch.py [--n 2000] [--reps 5] [--out profiles/train_epoch_h100.json]

For each workload (cavity 64x64 in fp32 and bf16 storage, tube 66x65) and batch size (8, 64, 256) it times one epoch
over N samples, without evaluation:
  * eager: DeviceFrames.loader + model(**batch) + loss["nmse"].backward() + FusedAdam.step() + zero_grad() + .item()
    per step;
  * graph: train_auto's epoch (cfdbench_b200.train._StepGraphs.epoch: upload of the permutation and the Adam table, one
    graph replay per step, the log copied back);
and, for context at B = 8, the reference's own loop: DataLoader + collate_fn (with its .cuda() copies) +
torch.optim.Adam on the same drop-in model.  Every time is a host clock around one epoch that ends in a device
synchronise; the implementations alternate, and the median of `--reps` repetitions is reported.  The card's name and
power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cfdbench_b200 import DeviceFrames, FusedAdam, synth  # noqa: E402
from cfdbench_b200.train import _StepGraphs, epoch_permutation  # noqa: E402
from test_gpu_eval_auto import _AutoSplit, _model  # noqa: E402


def _collate(batch):   # reference src/train_auto.py:33-58
    inputs, labels, case_params = zip(*batch)
    inputs, labels = torch.stack(inputs), torch.stack(labels)
    keys = [x for x in case_params[0].keys() if x not in ["rotated", "dx", "dy"]]
    cp = torch.tensor([[c[k] for k in keys] for c in case_params])
    return dict(inputs=inputs[:, :-1].cuda(), label=labels[:, :-1].cuda(), mask=inputs[:, -1:].cuda(), case_params=cp.cuda())


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", default="8,64,256")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "train_epoch_h100.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool times the GPU"
    card = _card()
    print("card:", card)
    rows = []
    for problem, act in (("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32")):
        ds = _AutoSplit(args.n, problem, seed=0)
        frames = DeviceFrames(ds, device="cuda")
        for b in (int(x) for x in args.batches.split(",")):
            m_e, m_g = _model(problem, act, seed=1), _model(problem, act, seed=1)
            opt_e = FusedAdam(m_e.parameters(), lr=1e-3)
            opt_g = FusedAdam(m_g.parameters(), lr=1e-3)
            graphs = _StepGraphs(m_g, frames, b, opt_g)
            gen_e, gen_g = torch.Generator().manual_seed(0), torch.Generator().manual_seed(0)
            state = dict(step=0)

            def eager():
                for batch in frames.loader(b, shuffle=True, generator=gen_e):
                    loss = m_e(**batch)["loss"]
                    loss["nmse"].backward()
                    opt_e.step()
                    opt_e.zero_grad()
                    loss["nmse"].item()
                torch.cuda.synchronize()

            def graph():
                graphs.epoch(epoch_permutation(args.n, b, gen_g), 1e-3, state["step"] + 1)
                state["step"] += graphs.steps
                torch.cuda.synchronize()

            impls = dict(eager=eager, graph=graph)
            if b == 8:
                m_r = _model(problem, act, seed=1)
                opt_r = torch.optim.Adam(m_r.parameters(), lr=1e-3)
                loader = torch.utils.data.DataLoader(ds, batch_size=b, shuffle=True, collate_fn=_collate)

                def reference():
                    for batch in loader:
                        loss = m_r(**batch)["loss"]
                        loss["nmse"].backward()
                        opt_r.step()
                        opt_r.zero_grad()
                        loss["nmse"].item()
                    torch.cuda.synchronize()
                impls["reference_loop"] = reference
            times = {k: [] for k in impls}
            for fn in impls.values():   # warm-up epoch of every implementation
                fn()
            for _ in range(args.reps):
                for k, fn in impls.items():
                    t0 = time.perf_counter()
                    fn()
                    times[k].append(time.perf_counter() - t0)
            del graphs
            steps = -(-args.n // b)
            med = {k: statistics.median(v) for k, v in times.items()}
            row = dict(problem=problem, grid=list(synth.grid(problem)), act_dtype=act, n=args.n, batch=b, steps=steps,
                       epoch_s={k: v for k, v in times.items()}, median_epoch_s=med,
                       median_step_ms={k: 1e3 * v / steps for k, v in med.items()},
                       speedup_graph_vs_eager=med["eager"] / med["graph"])
            if "reference_loop" in med:
                row["speedup_graph_vs_reference_loop"] = med["reference_loop"] / med["graph"]
            rows.append(row)
            print(json.dumps({k: row[k] for k in ("problem", "act_dtype", "batch", "median_step_ms",
                                                  "speedup_graph_vs_eager")}), flush=True)
            torch.cuda.empty_cache()
    rec = dict(tool="tools/time_train_epoch.py", card=card, torch=torch.__version__, reps=args.reps,
               timing="host clock around one epoch ending in torch.cuda.synchronize(); median of alternating reps",
               rows=rows)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
