"""Timing of the multi-step evaluation of a test split on this GPU.  The card name and power limit are read in the same run.

On one seeded synthetic split per configuration (`--cases` cases, `--steps` rollout steps, seeded drop-in Fno2d), two ways
to compute what the reference's `test_multistep.infer` returns (src/test_multistep.py:102-177):
  (a) the reference's loop, restated with the drop-in model: one B = 1 `generate_many` per case (graph-replayed), then
      for every step and case the masked-u `get_metrics` with its three `.item()` synchronisations, and the mean over
      cases;
  (b) `infer_multistep`: one B = n rollout per chunk of `--max-batch` cases, one metrics launch, one device-to-host copy.
Each is warmed up once (graph captures), then the two alternate for `--reps` repetitions; every repetition is timed
with a host clock that ends in a device synchronise.  The largest relative difference of the two results is reported.

    python tools/time_infer.py [--cases 100] [--steps 20] [--reps 5] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = (("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32"))


def per_case_loop(model, feats, cps, steps):
    """(a): the reference's infer, restated."""
    import numpy as np
    import torch
    with torch.no_grad():
        preds = [model.generate_many(inputs=f[0, :-1], case_params=c, mask=f[0, -1], steps=steps) for f, c in zip(feats, cps)]
    out = []
    for s in range(steps):
        rows = []
        for c, f in enumerate(feats):
            mask = f[s, -1]
            p, lab = preds[c][s][0][0] * mask, f[s, 0] * mask
            mse = ((p - lab) ** 2).mean().item()
            rows.append(dict(mse=mse, nmse=mse / (lab ** 2).mean().item(), mae=(p - lab).abs().mean().item()))
        out.append({k: float(np.mean([r[k] for r in rows])) for k in rows[0]})
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-batch", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    from cfdbench_b200 import Fno2d, infer_multistep, loss_name_to_fn, synth

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=60).stdout.strip() or "unknown"
    except Exception:  # noqa: BLE001
        power = "unknown"
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit=power, cases=args.cases, steps=args.steps,
               max_batch=args.max_batch, reps=args.reps, configs=[])
    for problem, act in CONFIGS:
        p = synth.n_case_params(problem)
        m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
                  modes1=12, modes2=12, act_dtype=act)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(1, n_params=p, spectral_gain=20.0).items()})
        m = m.cuda()
        feats_np, cps_np = synth.make_split(7, args.cases, problem, frames=(args.steps, args.steps + 5))
        feats = [torch.from_numpy(f).to(dev) for f in feats_np]
        cps = [torch.from_numpy(c).to(dev) for c in cps_np]

        def timed(fn):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            r = fn()
            torch.cuda.synchronize()
            return r, time.perf_counter() - t0
        run_a = lambda: per_case_loop(m, feats, cps, args.steps)                                    # noqa: E731
        run_b = lambda: infer_multistep(m, feats, cps, infer_steps=args.steps, max_batch=args.max_batch)  # noqa: E731
        ra, _ = timed(run_a)
        rb, _ = timed(run_b)
        ta, tb = [], []
        for _ in range(args.reps):
            ta.append(timed(run_a)[1])
            tb.append(timed(run_b)[1])
        diff = max(abs(x[k] - y[k]) / abs(y[k]) for x, y in zip(rb, ra) for k in y)
        row = dict(problem=problem, grid=list(synth.grid(problem)), act_dtype=act,
                   loop_s=dict(median=float(np.median(ta)), min=min(ta), max=max(ta)),
                   infer_multistep_s=dict(median=float(np.median(tb)), min=min(tb), max=max(tb)),
                   speedup_median=float(np.median(ta) / np.median(tb)), max_rel_diff=diff,
                   step0=rb[0], step_last=rb[-1])
        res["configs"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps({k: v for k, v in res.items() if k != "configs"}))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
