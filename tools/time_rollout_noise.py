"""Per-step time of `train_auto`'s graph-replayed K = 4 epochs with input noise on the start frame only against noise on
every rollout step (`noise_every_step=True`), on the same seeded chained split; plus the noise-stream kernel's own time.

    python tools/time_rollout_noise.py [--cases 20] [--frames 51] [--reps 5] [--out profiles/rollout_noise_h100.json]

For each workload (cavity 64x64 in fp32 and bf16 storage, tube 66x65) and batch size (8, 64, 256) it times one epoch
of four step graphs (_RolloutStepGraphs, input_noise_std = 0.01, without evaluation):
  * "K=4 G=1 start" / "K=4 G=1 every": pushforward, 3 inference steps and 1 trained step;
  * "K=4 G=4 start" / "K=4 G=4 every": full backpropagation through the 4 steps.
"every" adds one fno_add_input_noise_stream launch per rollout step after the first (3 per training step).  Each time
is a host clock around one epoch (upload, one graph replay per step, the log copied back) that ends in a device
synchronise; the four modes alternate, and the median of `--reps` repetitions is reported per step with the minimum and
maximum.  The stream kernel (input_noise_stream_kernel, out of place) is timed alone at B = 256 with CUDA events over
many launches.  The card's name, power limit and maximum SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cfdbench_b200 import DeviceFrames, FusedAdam, _lib, rollout_windows, synth  # noqa: E402
from cfdbench_b200.train import _RolloutStepGraphs, epoch_permutation  # noqa: E402
from test_gpu_eval_auto import _model  # noqa: E402
from test_gpu_train_rollout import _ChainSplit  # noqa: E402
from time_train_rollout_epoch import _card  # noqa: E402

SIGMA = 0.01
MODES = {"K=4 G=1 start": (4, 1, False), "K=4 G=1 every": (4, 1, True), "K=4 G=4 start": (4, 4, False),
         "K=4 G=4 every": (4, 4, True)}


def _stream_kernel_us(frames: DeviceFrames, b: int, launches: int) -> float:
    """Mean time of one out-of-place fno_add_input_noise_stream launch on b frames (CUDA events, `launches` launches)."""
    lib = _lib.load()
    bt = frames.batch(torch.arange(b) % frames.n)
    out = torch.empty_like(bt["inputs"])
    idx = (torch.arange(b) % frames.n).cuda()
    base = torch.ones(1, dtype=torch.int64, device="cuda")
    off = torch.zeros(1, dtype=torch.int32, device="cuda")
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def launch():
        _lib.check(lib.fno_add_input_noise_stream(bt["inputs"].data_ptr(), out.data_ptr(), bt["mask"].data_ptr(),
                                                  idx.data_ptr(), b, frames.height, frames.width, SIGMA, 1,
                                                  base.data_ptr(), off.data_ptr(), 2, st), "fno_add_input_noise_stream")
    for _ in range(20):
        launch()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        launch()
    e1.record()
    torch.cuda.synchronize()
    return 1e3 * e0.elapsed_time(e1) / launches


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=20)
    ap.add_argument("--frames", type=int, default=51, help="frames per case (samples per case = frames - 1)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--batches", default="8,64,256")
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "rollout_noise_h100.json"))
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this tool times the GPU"
    card = _card()
    print("card:", card)
    rows, kernel = [], []
    for problem, act in (("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32")):
        ds = _ChainSplit([args.frames] * args.cases, problem, s=1, seed=0)
        frames = DeviceFrames(ds, device="cuda")
        if act == "float32":
            us = _stream_kernel_us(frames, 256, args.launches)
            n_el = 256 * 2 * frames.height * frames.width
            kernel.append(dict(problem=problem, grid=list(synth.grid(problem)), batch=256, launches=args.launches,
                               mean_us=us, elements=n_el,
                               effective_gb_per_s=(n_el * 8 + n_el // 2 * 4) / us / 1e3))   # in read, out written, mask
            print(json.dumps(kernel[-1]), flush=True)
        for b in (int(x) for x in args.batches.split(",")):
            impls, state = {}, {}
            for name, (K, G, every) in MODES.items():
                m = _model(problem, act, seed=1)
                opt = FusedAdam(m.parameters(), lr=1e-3)
                windows = rollout_windows(ds.case_ids, K, 1)
                graphs = _RolloutStepGraphs(m, frames, b, opt, windows.size, K, 1, G, noise_std=SIGMA, noise_seed=1,
                                            noise_every_step=every)
                state[name] = dict(graphs=graphs, windows=windows, gen=torch.Generator().manual_seed(0), step=0)

                def run(s=state[name]):
                    w = s["windows"]
                    s["graphs"].epoch(w[epoch_permutation(w.size, b, s["gen"])], 1e-3, s["step"] + 1)
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
            steps = {k: state[k]["graphs"].steps for k in impls}
            med = {k: statistics.median(v) for k, v in times.items()}
            row = dict(problem=problem, grid=list(synth.grid(problem)), act_dtype=act, batch=b, steps=steps,
                       epoch_s=times, spread_step_ms={k: [1e3 * min(v) / steps[k], 1e3 * max(v) / steps[k]]
                                                      for k, v in times.items()},
                       median_step_ms={k: 1e3 * v / steps[k] for k, v in med.items()},
                       every_over_start={g: med[f"K=4 {g} every"] / med[f"K=4 {g} start"] for g in ("G=1", "G=4")})
            rows.append(row)
            print(json.dumps({k: row[k] for k in ("problem", "act_dtype", "batch", "median_step_ms", "every_over_start")}),
                  flush=True)
            del impls, state
            torch.cuda.empty_cache()
    rec = dict(tool="tools/time_rollout_noise.py", card=card, torch=torch.__version__, reps=args.reps,
               split=dict(cases=args.cases, frames_per_case=args.frames, time_step_size=1),
               modes={k: dict(rollout_steps=v[0], rollout_grad_steps=v[1], input_noise_std=SIGMA, noise_every_step=v[2])
                      for k, v in MODES.items()},
               timing="host clock around one epoch ending in torch.cuda.synchronize(), divided by the epoch's steps; "
                      "median of alternating reps, spread = [min, max]; stream kernel: CUDA events around many launches",
               stream_kernel=kernel, rows=rows)
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, "w") as f:
        json.dump(rec, f, indent=1)
    print("wrote", args.out)


if __name__ == "__main__":
    main()
