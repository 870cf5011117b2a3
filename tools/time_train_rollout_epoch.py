"""Epoch time of `train_auto(rollout_steps=K)`'s graph-replayed steps against the eager rollout-training loop a user
writes with the drop-in pieces, on the same seeded chained split.

    python tools/time_train_rollout_epoch.py [--cases 20] [--frames 51] [--reps 5] \
        [--out profiles/train_rollout_epoch_h100.json]

For each workload (cavity 64x64 in fp32 and bf16 storage, tube 66x65), rollout length K (1, 4, 8) and batch size
(8, 64, 256) it times one epoch over the split's K-step windows, without evaluation:
  * eager: per step DeviceFrames.rollout_batch + Fno2d.rollout + sum(nmse_k) / K + backward() + FusedAdam.step() +
    zero_grad() + .item();
  * graph: train_auto's epoch (cfdbench_b200.train._RolloutStepGraphs.epoch, _StepGraphs.epoch for K = 1: upload of the
    permutation and the Adam table, one graph replay per step, the log copied back).
Every time is a host clock around one epoch that ends in a device synchronise; the two implementations alternate, and
the median of `--reps` repetitions is reported with the minimum and maximum.  The card's name and power limit are read
in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from cfdbench_b200 import DeviceFrames, FusedAdam, rollout_windows, synth  # noqa: E402
from cfdbench_b200.data import index_batches  # noqa: E402
from cfdbench_b200.train import _RolloutStepGraphs, _StepGraphs, epoch_permutation  # noqa: E402
from test_gpu_eval_auto import _model  # noqa: E402
from test_gpu_train_rollout import _ChainSplit  # noqa: E402


def _card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=20)
    ap.add_argument("--frames", type=int, default=51, help="frames per case (samples per case = frames - 1)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", default="1,4,8")
    ap.add_argument("--batches", default="8,64,256")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "train_rollout_epoch_h100.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool times the GPU"
    card = _card()
    print("card:", card)
    rows = []
    for problem, act in (("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32")):
        ds = _ChainSplit([args.frames] * args.cases, problem, s=1, seed=0)
        frames = DeviceFrames(ds, device="cuda")
        for K in (int(x) for x in args.steps.split(",")):
            windows = rollout_windows(ds.case_ids, K, 1)
            for b in (int(x) for x in args.batches.split(",")):
                m_e, m_g = _model(problem, act, seed=1), _model(problem, act, seed=1)
                opt_e = FusedAdam(m_e.parameters(), lr=1e-3)
                opt_g = FusedAdam(m_g.parameters(), lr=1e-3)
                if K == 1:
                    graphs = _StepGraphs(m_g, frames, b, opt_g)
                else:
                    graphs = _RolloutStepGraphs(m_g, frames, b, opt_g, windows.size, K, 1)
                gen_e, gen_g = torch.Generator().manual_seed(0), torch.Generator().manual_seed(0)
                state = dict(step=0)

                def eager():
                    for ib in index_batches(windows.size, b, True, gen_e):
                        bt = frames.rollout_batch(windows[ib], K)
                        preds = m_e.rollout(bt["inputs"], bt["case_params"], bt["mask"], K)
                        loss = sum(m_e.loss_fn(preds=preds[k], labels=bt["labels"][k])["nmse"] for k in range(K)) / K
                        loss.backward()
                        opt_e.step()
                        opt_e.zero_grad()
                        loss.item()
                    torch.cuda.synchronize()

                def graph():
                    graphs.epoch(windows[epoch_permutation(windows.size, b, gen_g)], 1e-3, state["step"] + 1)
                    state["step"] += graphs.steps
                    torch.cuda.synchronize()

                impls = dict(eager=eager, graph=graph)
                times = {k: [] for k in impls}
                for fn in impls.values():   # warm-up epoch of every implementation
                    fn()
                for _ in range(args.reps):
                    for k, fn in impls.items():
                        t0 = time.perf_counter()
                        fn()
                        times[k].append(time.perf_counter() - t0)
                del graphs
                steps = -(-windows.size // b)
                med = {k: statistics.median(v) for k, v in times.items()}
                row = dict(problem=problem, grid=list(synth.grid(problem)), act_dtype=act, rollout_steps=K,
                           windows=int(windows.size), batch=b, steps=steps, epoch_s=times, median_epoch_s=med,
                           spread_epoch_s={k: [min(v), max(v)] for k, v in times.items()},
                           median_step_ms={k: 1e3 * v / steps for k, v in med.items()},
                           speedup_graph_vs_eager=med["eager"] / med["graph"])
                rows.append(row)
                print(json.dumps({k: row[k] for k in ("problem", "act_dtype", "rollout_steps", "batch", "median_step_ms",
                                                      "speedup_graph_vs_eager")}), flush=True)
                del m_e, m_g, opt_e, opt_g
                torch.cuda.empty_cache()
    rec = dict(tool="tools/time_train_rollout_epoch.py", card=card, torch=torch.__version__, reps=args.reps,
               split=dict(cases=args.cases, frames_per_case=args.frames, time_step_size=1),
               timing="host clock around one epoch ending in torch.cuda.synchronize(); median of alternating reps, "
                      "spread = [min, max]",
               rows=rows)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
