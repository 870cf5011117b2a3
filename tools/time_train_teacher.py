"""Per-step time of `train_auto`'s graph-replayed K-step rollout epochs with teacher forcing (`teacher_forcing=0.5`)
against the free rollout (`teacher_forcing=None`), on the same seeded chained split; plus each mode's graph-capture
time and peak allocated memory.

    python tools/time_train_teacher.py [--cases 20] [--frames 51] [--reps 5] [--out profiles/train_teacher_h100.json]

For each workload (cavity 64x64 in fp32 and bf16 storage, tube 66x65) and batch size (8, 64, 256) at K = 4 it builds
the step graphs of two modes (_RolloutStepGraphs, as train_auto builds them):
  * "free": every rollout step is fed the previous prediction;
  * "teacher": the step draws its flags (fno_teacher_flags, p = 0.5) and every step s >= 1 is fed a frame chosen by
    them (one feed launch per step); the sweep's hand-offs are gated by the flags.
The graph-capture time is a host clock around the construction ending in a device synchronise.  The peak allocated
memory is torch.cuda.max_memory_allocated over the construction and one epoch, above what was allocated before.  The
per-step time is a host clock around one epoch without evaluation (uploads, one graph replay per step, the log copied
back) ending in a device synchronise; the modes alternate, and the median of `--reps` repetitions is reported per step
with the minimum and maximum.  Both modes visit the same windows in the same orders.  The card's name, power limit and
maximum SM clock are read in the same run.
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

from cfdbench_b200 import DeviceFrames, FusedAdam, rollout_windows, synth  # noqa: E402
from cfdbench_b200.train import _RolloutStepGraphs, epoch_permutation  # noqa: E402
from test_gpu_eval_auto import _model  # noqa: E402
from test_gpu_train_rollout import _ChainSplit  # noqa: E402
from time_train_rollout_epoch import _card  # noqa: E402

K = 4
P = 0.5
MODES = ("free", "teacher")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=20)
    ap.add_argument("--frames", type=int, default=51, help="frames per case (samples per case = frames - 1)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", default="8,64,256")
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "train_teacher_h100.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool times the GPU"
    card = _card()
    print("card:", card)
    rows = []
    for problem, act in (("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32")):
        ds = _ChainSplit([args.frames] * args.cases, problem, s=1, seed=0)
        frames = DeviceFrames(ds, device="cuda")
        windows = rollout_windows(ds.case_ids, K, 1)
        for b in (int(x) for x in args.batches.split(",")):
            state, capture_s, peak = {}, {}, {}
            for name in MODES:
                m = _model(problem, act, seed=1)
                opt = FusedAdam(m.parameters(), lr=1e-3)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                t0 = time.perf_counter()
                graphs = _RolloutStepGraphs(m, frames, b, opt, windows.size, K, 1, K, teacher=name == "teacher",
                                            teacher_seed=0)
                torch.cuda.synchronize()
                capture_s[name] = time.perf_counter() - t0
                s = state[name] = dict(graphs=graphs, gen=torch.Generator().manual_seed(0), step=0, model=m)

                def run(s=s, teacher=name == "teacher"):
                    perm = windows[epoch_permutation(windows.size, b, s["gen"])]
                    if teacher:
                        s["graphs"].epoch(perm, 1e-3, s["step"] + 1, teacher_prob=P)
                    else:
                        s["graphs"].epoch(perm, 1e-3, s["step"] + 1)
                    s["step"] += s["graphs"].steps
                    torch.cuda.synchronize()
                s["run"] = run
                run()   # warm-up epoch, inside the peak-memory window
                peak[name] = torch.cuda.max_memory_allocated() - base
            times = {k: [] for k in MODES}
            for _ in range(args.reps):
                for k in MODES:
                    t0 = time.perf_counter()
                    state[k]["run"]()
                    times[k].append(time.perf_counter() - t0)
            steps = state["free"]["graphs"].steps
            med = {k: statistics.median(v) for k, v in times.items()}
            row = dict(problem=problem, grid=list(synth.grid(problem)), act_dtype=act, K=K, p=P, batch=b,
                       steps_per_epoch=steps, epoch_s=times,
                       median_step_ms={k: 1e3 * v / steps for k, v in med.items()},
                       spread_step_ms={k: [1e3 * min(v) / steps, 1e3 * max(v) / steps] for k, v in times.items()},
                       teacher_over_free=med["teacher"] / med["free"], capture_s=capture_s,
                       peak_allocated_bytes=peak)
            rows.append(row)
            print(json.dumps({k: row[k] for k in ("problem", "act_dtype", "batch", "median_step_ms",
                                                  "teacher_over_free", "peak_allocated_bytes")}), flush=True)
            del state
            torch.cuda.empty_cache()
    rec = dict(tool="tools/time_train_teacher.py", card=card, torch=torch.__version__, reps=args.reps,
               split=dict(cases=args.cases, frames_per_case=args.frames, time_step_size=1),
               modes=dict(free="teacher_forcing=None", teacher=f"teacher_forcing={P}"),
               timing="host clock around one epoch ending in torch.cuda.synchronize(), divided by the epoch's steps; "
                      "median of alternating reps, spread = [min, max]; capture: host clock around the step graphs' "
                      "construction ending in torch.cuda.synchronize(); peak: max_memory_allocated over construction "
                      "and one epoch minus memory_allocated before",
               rows=rows)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
