"""Training through a K-step rollout: chained `generate` under autograd vs `Fno2d.rollout` (one reused saved set, the
backward recomputes each step's activations).  Per case (grid, storage, K) and path: the time of one training step --
rollout forward, an mse loss over the K predictions, backward, FusedAdam step -- (CUDA events around `--iters` steps,
median of `--reps` repetitions after `--warmup` steps) and the peak allocated memory of one step from a cold model.
The largest K that fits is extrapolated from the two measured peaks (linear in K) and the card's total memory.
The card name and power limit are read in the same run and printed first; one JSON line per case is printed and
appended to `--out` when given.

    python tools/time_rollout_train.py [--batch 256] [--steps 4,20] [--out profiles/rollout_train_h100.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", default="4,20")
    ap.add_argument("--cases", default="cavity:bfloat16,cavity:float32,tube:float32")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import numpy as np
    import torch
    from cfdbench_b200 import Fno2d, FusedAdam, loss_name_to_fn, synth

    if not torch.cuda.is_available():
        raise SystemExit("time_rollout_train.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=60).stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    card = torch.cuda.get_device_name(dev)
    total = torch.cuda.get_device_properties(dev).total_memory
    print(f"# {card}, power limit {power}, {total / 2**30:.1f} GiB; B={args.batch}; median of {args.reps} x "
          f"{args.iters} training steps", flush=True)

    b, p = args.batch, 5
    ks = [int(k) for k in args.steps.split(",")]
    sd = synth.make_state_dict(0, n_params=p, spectral_gain=50.0)
    for case in args.cases.split(","):
        where, act = case.split(":")
        bt = {k: torch.from_numpy(v).to(dev) for k, v in synth.make_batch(1, b, where).items()}
        gh, gw = bt["inputs"].shape[-2:]
        m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
                  modes1=12, modes2=12, act_dtype=act)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
        opt = FusedAdam(m.parameters(), lr=1e-6)
        res = {"card": card, "power_limit": power, "grid": f"{gh}x{gw}", "act_dtype": act, "batch": b}
        for path in ("chained", "rollout"):
            peaks = {}
            for k in ks:
                labels = torch.randn(k, b, 2, gh, gw, device=dev)

                def step():
                    if path == "rollout":
                        seq = m.rollout(bt["inputs"], bt["case_params"], bt["mask"], k)
                    else:
                        x, preds = bt["inputs"], []
                        for _ in range(k):
                            x = m.generate(x, bt["case_params"], bt["mask"])
                            preds.append(x)
                        seq = torch.stack(preds)
                    loss = ((seq - labels) ** 2).mean()
                    opt.zero_grad(set_to_none=True)
                    loss.backward()
                    opt.step()

                m.invalidate_packed()
                torch.cuda.synchronize(dev)
                torch.cuda.empty_cache()
                torch.cuda.reset_peak_memory_stats(dev)
                base = torch.cuda.memory_allocated(dev)
                step()
                torch.cuda.synchronize(dev)
                peaks[k] = torch.cuda.max_memory_allocated(dev) - base
                for _ in range(args.warmup):
                    step()
                torch.cuda.synchronize(dev)
                ts = []
                for _ in range(args.reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(args.iters):
                        step()
                    e1.record()
                    e1.synchronize()
                    ts.append(e0.elapsed_time(e1) / args.iters)
                res[f"{path}_K{k}_ms"] = round(float(np.median(ts)), 3)
                res[f"{path}_K{k}_ms_spread"] = [round(min(ts), 3), round(max(ts), 3)]
                res[f"{path}_K{k}_peak_GB"] = round(peaks[k] / 1e9, 3)
                del labels
            k0, k1 = ks[0], ks[-1]
            if k1 > k0:
                per_step = (peaks[k1] - peaks[k0]) / (k1 - k0)
                res[f"{path}_MB_per_step"] = round(per_step / 1e6, 2)
                res[f"{path}_max_K_fit"] = int(k0 + (total - torch.cuda.memory_allocated(dev) - peaks[k0]) // max(per_step, 1))
        line = json.dumps(res)
        print(line, flush=True)
        if args.out:
            os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
            with open(args.out, "a") as f:
                f.write(line + "\n")
        del m, opt, bt
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
