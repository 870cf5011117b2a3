"""Timing of checkpoint selection by rollout error on this GPU.  The card name, power limit and max SM clock are read in
the same run.

On one seeded, chained synthetic dev split per configuration (`--cases` cases of `--frames` frames: inputs =
frames[:-1], labels = frames[1:], about 2,000 samples at the defaults; synth's fields and masks; seeded drop-in Fno2d
with the nmse loss), three ways to compute the S-step rollout error of every window (S = `--steps`):
  (a) `evaluate_rollout_auto(model, frames, S)` (the chain check included);
  (b) the eager loop a user writes today: per chunk of `--max-batch` windows `DeviceFrames.batch` of the starts,
      `torch.stack(generate_many(...))`, S label gathers stacked into (S, B, H, W), the start mask expanded, and
      `multistep_metrics`;
  (c) the reference-style loop: one B = 1 `generate_many` per window and three `.item()` calls per step.
Each is warmed up once, then they alternate for `--reps` repetitions, each timed with a host clock that ends in a
device synchronise; the medians are reported.  Then one `train_auto` epoch plus its evaluation (a train split like the
dev split, batch 32) with and without `dev_rollout_steps=S`, alternating likewise; each call captures its step graphs.

    python tools/time_dev_rollout.py [--cases 20] [--frames 101] [--steps 20] [--reps 5] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = (("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32"))


class ChainedSplit:
    """`.inputs`, `.labels` (N, 3, H, W), `.case_ids`, `.case_params` and `.time_step_size` = 1 as the reference's auto
    datasets have them: per case `frames` frames of synth's clipped-normal fields under the problem's mask,
    inputs = frames[:-1], labels = frames[1:]."""

    def __init__(self, n_cases, frames, problem, seed=0):
        import numpy as np
        import torch
        from cfdbench_b200 import synth
        rng = np.random.default_rng(seed)
        gh, gw = synth.grid(problem)
        masks = synth.make_mask(rng, n_cases, problem)[:, 0]
        ins, labs, ids = [], [], []
        for c in range(n_cases):
            fr = np.empty((frames, 3, gh, gw), np.float32)
            fr[:, :2] = np.clip(rng.standard_normal((frames, 2, gh, gw)), -3, 3)
            fr[:, 2] = masks[c]
            ins.append(fr[:-1])
            labs.append(fr[1:])
            ids += [c] * (frames - 1)
        self.inputs, self.labels = torch.from_numpy(np.concatenate(ins)), torch.from_numpy(np.concatenate(labs))
        self.case_ids = np.asarray(ids)
        self.time_step_size = 1
        p = synth.n_case_params(problem)
        self.case_params = [{f"p{j}": float(rng.standard_normal()) for j in range(p)} for _ in range(n_cases)]

    def __len__(self):
        return len(self.inputs)


def eager_loop(model, frames, windows, steps, max_batch):
    """(b): the composition of existing pieces, one multistep_metrics call (one synchronisation) per chunk."""
    import numpy as np
    import torch
    from cfdbench_b200.metrics import multistep_metrics
    per_step = [dict(mse=0.0, nmse=0.0, mae=0.0) for _ in range(steps)]
    with torch.no_grad():
        for lo in range(0, windows.size, max_batch):
            starts = torch.from_numpy(windows[lo:lo + max_batch])
            b0 = frames.batch(starts)
            preds = torch.stack(model.generate_many(b0["inputs"], b0["case_params"], b0["mask"], steps))
            label_u = torch.stack([frames.batch(starts + k)["label"][:, 0] for k in range(steps)])
            mask = b0["mask"][:, 0].expand(steps, -1, -1, -1).contiguous()
            res = multistep_metrics(preds, label_u, mask)
            for k in range(steps):
                for name in per_step[k]:
                    per_step[k][name] += res[k][name] * starts.numel()
    rows = [{k: v / windows.size for k, v in r.items()} for r in per_step]
    return dict(steps=rows, loss=float(np.mean([r["nmse"] for r in rows])))


def reference_loop(model, frames, windows, steps):
    """(c): one B = 1 rollout per window and get_metrics' three .item() calls per step (reference
    src/test_multistep.py:73-83, 102-132), targets frames_out[j + k]."""
    import numpy as np
    import torch
    per_step = [dict(mse=0.0, nmse=0.0, mae=0.0) for _ in range(steps)]
    fout = frames.frames_out
    with torch.no_grad():
        for j in windows.tolist():
            b0 = frames.batch([j])
            preds = model.generate_many(b0["inputs"], b0["case_params"], b0["mask"], steps)
            m = b0["mask"][:, 0]
            for k in range(steps):
                p = preds[k][:, 0] * m
                lab = fout[j + k, 0].float()[None] * m
                mse = ((p - lab) ** 2).mean().item()
                nmse = mse / (lab ** 2).mean().item()
                mae = (p - lab).abs().mean().item()
                per_step[k]["mse"] += mse
                per_step[k]["nmse"] += nmse
                per_step[k]["mae"] += mae
    rows = [{k: v / windows.size for k, v in r.items()} for r in per_step]
    return dict(steps=rows, loss=float(np.mean([r["nmse"] for r in rows])))


def card_info():
    out = {}
    for key, q in (("power_limit", "power.limit"), ("max_sm_clock", "clocks.max.sm")):
        try:
            out[key] = subprocess.run(["nvidia-smi", "--id=0", f"--query-gpu={q}", "--format=csv,noheader"],
                                      capture_output=True, text=True, timeout=60).stdout.strip() or "unknown"
        except Exception:  # noqa: BLE001
            out[key] = "unknown"
    return out


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", type=int, default=20)
    ap.add_argument("--frames", type=int, default=101)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-batch", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    from cfdbench_b200 import DeviceFrames, Fno2d, evaluate_rollout_auto, loss_name_to_fn, rollout_windows, synth, train_auto

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    S = args.steps
    res = dict(gpu=torch.cuda.get_device_name(dev), **card_info(), cases=args.cases, frames_per_case=args.frames,
               samples=args.cases * (args.frames - 1), steps=S, max_batch=args.max_batch, reps=args.reps, configs=[])
    print(json.dumps({k: v for k, v in res.items() if k != "configs"}), flush=True)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return r, time.perf_counter() - t0

    def alternate(runs):
        first = {k: timed(f)[0] for k, f in runs.items()}   # warm-up
        times = {k: [] for k in runs}
        for _ in range(args.reps):
            for k, f in runs.items():
                times[k].append(timed(f)[1])
        return first, {k: dict(median=float(np.median(v)), min=min(v), max=max(v)) for k, v in times.items()}

    def make_model(problem, act):
        p = synth.n_case_params(problem)
        m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
                  modes1=12, modes2=12, act_dtype=act)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(1, n_params=p, spectral_gain=20.0).items()})
        return m.cuda()

    for problem, act in CONFIGS:
        m = make_model(problem, act)
        ds = ChainedSplit(args.cases, args.frames, problem, seed=7)
        frames = DeviceFrames(ds, device=dev)
        windows = rollout_windows(ds.case_ids, S, 1)
        first, times = alternate(dict(
            evaluate_rollout_auto=lambda: evaluate_rollout_auto(m, frames, S, max_batch=args.max_batch),  # noqa: E731
            eager_loop=lambda: eager_loop(m, frames, windows, S, args.max_batch),                            # noqa: E731
            reference_loop=lambda: reference_loop(m, frames, windows, S)))                                    # noqa: E731
        ours = first["evaluate_rollout_auto"]
        diff = {k: max(abs(a["nmse"] - b["nmse"]) / abs(b["nmse"]) for a, b in zip(ours["steps"], first[k]["steps"]))
                for k in ("eager_loop", "reference_loop")}
        row = dict(problem=problem, grid=list(synth.grid(problem)), act_dtype=act, windows=int(windows.size),
                   **{f"{k}_s": v for k, v in times.items()},
                   speedup_vs_eager=times["eager_loop"]["median"] / times["evaluate_rollout_auto"]["median"],
                   speedup_vs_reference=times["reference_loop"]["median"] / times["evaluate_rollout_auto"]["median"],
                   max_rel_step_nmse_diff=diff, loss=ours["loss"])
        # one train_auto epoch plus its evaluation, with and without checkpoint selection by rollout error
        tr = DeviceFrames(ChainedSplit(args.cases, args.frames, problem, seed=8), device=dev)
        with tempfile.TemporaryDirectory() as tmp:
            def epoch(opt):
                mm = make_model(problem, act)
                return train_auto(mm, tr, frames, os.path.join(tmp, str(opt)), num_epochs=1, batch_size=32,
                                  eval_batch_size=16, log_interval=10 ** 9, eval_interval=1,
                                  generator=torch.Generator().manual_seed(0), dev_rollout_steps=opt)
            _, ep_times = alternate(dict(train_epoch_single_step_dev=lambda: epoch(None),      # noqa: E731
                                         train_epoch_dev_rollout=lambda: epoch(S)))             # noqa: E731
        row.update({f"{k}_s": v for k, v in ep_times.items()})
        res["configs"].append(row)
        print(json.dumps(row), flush=True)
        del frames, tr
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
