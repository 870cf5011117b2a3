"""Cost of Fno2d's input gradients on this GPU: cavity, B=256, fp32 and bf16 storage, CUDA events around `--iters`
calls, median of `--reps` repetitions (after `--warmup` calls).  Cases:
  (a) forward + nmse.backward(), parameter gradients only (the train_auto.py step without the optimizer)
  (b) the same, also differentiating w.r.t. inputs and case_params
  (c) frozen model (no parameter requires grad): forward + data-only backward to inputs and case_params
  (d) one 4-step unrolled training step: x_{k+1} = forward(x_k), nmse against label_k summed over the steps, one backward
The card name and power limit are read in the same run and printed first.

    python tools/time_input_grads.py [--batch 256] [--cases abcd] [--tree DIR]

--tree DIR times the package of another checkout (e.g. the previous commit, built in place) -- case (a) exists there too.
"""
import argparse
import os
import subprocess
import sys


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--cases", default="abcd")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tree", default=None)
    args = ap.parse_args()
    root = os.path.abspath(args.tree) if args.tree else os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    import numpy as np
    import torch
    from cfdbench_b200 import Fno2d, loss_name_to_fn, synth

    if not torch.cuda.is_available():
        raise SystemExit("time_input_grads.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=60).stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    print(f"# {torch.cuda.get_device_name(dev)}, power limit {power}; tree {root}; cavity B={args.batch}; "
          f"median of {args.reps} x {args.iters} calls", flush=True)

    p, unroll = 5, 4
    sd = synth.make_state_dict(0, n_params=p, spectral_gain=50.0)
    batch = synth.make_batch(1, args.batch, "cavity")
    tb = {k: torch.from_numpy(v).to(dev) for k, v in batch.items()}
    labels = [torch.from_numpy(synth.make_batch(2 + k, args.batch, "cavity")["label"]).to(dev) for k in range(unroll)]

    def model(act, frozen=False):
        m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
                  modes1=12, modes2=12, act_dtype=act)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
        for prm in m.parameters():
            prm.requires_grad_(not frozen)
        return m

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize(dev)
        ts = []
        for _ in range(args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.iters):
                fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) / args.iters)
        return float(np.median(ts)), ts

    for act in ("float32", "bfloat16"):
        m, mf = model(act), model(act, frozen=True)

        def step(mod, with_inputs, steps=1):
            mod.zero_grad(set_to_none=True)
            x = tb["inputs"].detach().requires_grad_(with_inputs)
            cp = tb["case_params"].detach().requires_grad_(with_inputs)
            cur, loss = x, 0.0
            for k in range(steps):
                out = mod(inputs=cur, case_params=cp, mask=tb["mask"], label=labels[k] if steps > 1 else tb["label"])
                cur, loss = out["preds"], loss + out["loss"]["nmse"]
            loss.backward()

        cases = {
            "a": ("fwd + bwd, parameter gradients", lambda: step(m, False)),
            "b": ("fwd + bwd, parameter + input / case_params gradients", lambda: step(m, True)),
            "c": ("fwd + data-only bwd, frozen model", lambda: step(mf, True)),
            "d": (f"{unroll}-step unrolled fwd + bwd, parameter gradients", lambda: step(m, False, unroll)),
        }
        for key in args.cases:
            what, fn = cases[key]
            med, ts = timed(fn)
            print(f"{act:8s} ({key}) {what:55s} {med:8.3f} ms  (reps: {', '.join(f'{t:.3f}' for t in ts)})", flush=True)
        del m, mf
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
