"""Timing of the single-step evaluation of a split on this GPU.  The card name and power limit are read in the same run.

On one seeded synthetic split per configuration (`--samples` samples built from `synth`'s fields and masks, seeded
drop-in Fno2d with the nmse loss), two ways to compute what the reference's `train_auto.evaluate` returns
(src/train_auto.py:61-148), without its plots:
  (a) the reference's loop, restated with the drop-in model: `DataLoader` + collate_fn (restated) + `.cuda()`, the input
      loss, `model(**batch)`, `.cpu().tolist()` of every score and `preds.cpu()` per batch;
  (b) `evaluate_auto`, once from the dataset object (uploaded by the call) and once from a `DeviceFrames` built
      beforehand (the dev split reused across evaluation intervals).
Both at batch_size 1 (what `test()` uses) and 16 (the default `eval_batch_size` of the dev evaluation).  Each is warmed
up once, then they alternate for `--reps` repetitions; every repetition is timed with a host clock that ends in a device
synchronise.  The largest relative difference of the scores and whether the predictions are equal are reported.

    python tools/time_eval.py [--samples 2000] [--reps 5] [--max-batch 256] [--out FILE.json]
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = (("cavity", "float32"), ("cavity", "bfloat16"), ("tube", "float32"))
EXCLUDED = ("rotated", "dx", "dy")


class AutoSplit:
    """`.inputs`, `.labels` (N, 3, H, W), `.case_ids`, `.case_params` and `__getitem__` as the reference's auto datasets
    have them, filled with synth's clipped-normal fields and the problem's masks."""

    def __init__(self, n, problem, seed=0, n_cases=20):
        import numpy as np
        import torch
        from cfdbench_b200 import synth
        rng = np.random.default_rng(seed)
        gh, gw = synth.grid(problem)
        mask = synth.make_mask(rng, n, problem)[:, 0]
        ins = np.empty((n, 3, gh, gw), np.float32)
        labs = np.empty((n, 3, gh, gw), np.float32)
        for a in (ins, labs):
            a[:, :2] = np.clip(rng.standard_normal((n, 2, gh, gw)), -3, 3)
            a[:, 2] = mask
        self.inputs, self.labels = torch.from_numpy(ins), torch.from_numpy(labs)
        self.case_ids = np.sort(rng.integers(0, n_cases, n))
        p = synth.n_case_params(problem)
        self.case_params = [dict(rotated=0, **{f"p{j}": float(rng.standard_normal()) for j in range(p)})
                            for _ in range(n_cases)]

    def __len__(self):
        return len(self.inputs)

    def __getitem__(self, idx):
        return self.inputs[idx], self.labels[idx], self.case_params[self.case_ids[idx]]


def collate(batch):
    """The reference's collate_fn (src/train_auto.py:33-58), restated."""
    import torch
    inputs, labels, case_params = zip(*batch)
    inputs, labels = torch.stack(inputs), torch.stack(labels)
    keys = [k for k in case_params[0] if k not in EXCLUDED]
    cp = torch.tensor([[c[k] for k in keys] for c in case_params])
    return dict(inputs=inputs[:, :-1].cuda(), label=labels[:, :-1].cuda(), mask=inputs[:, -1:].cuda(), case_params=cp.cuda())


def reference_loop(model, ds, batch_size):
    """(a): the reference's evaluate, restated without plots."""
    import numpy as np
    import torch
    loader = torch.utils.data.DataLoader(ds, batch_size=batch_size, shuffle=False, collate_fn=collate)
    scores = {k: [] for k in model.loss_fn.get_score_names()}
    input_scores = copy.deepcopy(scores)
    all_preds = []
    model.eval()
    with torch.inference_mode():
        for batch in loader:
            inputs, labels = batch["inputs"], batch["label"]
            input_loss = model.loss_fn(labels=labels[:, :1], preds=inputs[:, :1])
            for k in input_scores:
                input_scores[k].append(input_loss[k].cpu().tolist())
            out = model(**batch)
            preds = out["preds"].view(-1, 1, *labels.shape[2:])
            for k in scores:
                scores[k].append(out["loss"][k].cpu().tolist())
            all_preds.append(preds.cpu())
    mean = {}
    for k in scores:
        mean[k] = float(np.mean(scores[k]))
        mean[f"input_{k}"] = float(np.mean(input_scores[k]))
    return dict(preds=torch.cat(all_preds), scores=dict(mean=mean, all=scores))


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--samples", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--max-batch", type=int, default=256)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import numpy as np
    import torch
    from cfdbench_b200 import DeviceFrames, Fno2d, evaluate_auto, loss_name_to_fn, synth

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=60).stdout.strip() or "unknown"
    except Exception:  # noqa: BLE001
        power = "unknown"
    res = dict(gpu=torch.cuda.get_device_name(dev), power_limit=power, samples=args.samples, max_batch=args.max_batch,
               reps=args.reps, configs=[])
    print(json.dumps({k: v for k, v in res.items() if k != "configs"}), flush=True)

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return r, time.perf_counter() - t0

    def stats(ts):
        return dict(median=float(np.median(ts)), min=min(ts), max=max(ts))

    for problem, act in CONFIGS:
        p = synth.n_case_params(problem)
        m = Fno2d(in_chan=2, out_chan=2, n_case_params=p, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
                  modes1=12, modes2=12, act_dtype=act)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in synth.make_state_dict(1, n_params=p, spectral_gain=20.0).items()})
        m = m.cuda()
        ds = AutoSplit(args.samples, problem, seed=7)
        frames = DeviceFrames(ds, device=dev)
        for bs in (1, 16):
            runs = dict(
                loop=lambda: reference_loop(m, ds, bs),                                                  # noqa: E731
                evaluate_auto_dataset=lambda: evaluate_auto(m, ds, batch_size=bs, max_batch=args.max_batch),  # noqa: E731
                evaluate_auto_frames=lambda: evaluate_auto(m, frames, batch_size=bs, max_batch=args.max_batch))  # noqa: E731
            first = {k: timed(f)[0] for k, f in runs.items()}
            times = {k: [] for k in runs}
            for _ in range(args.reps):
                for k, f in runs.items():
                    times[k].append(timed(f)[1])
            ref = first["loop"]
            ours = first["evaluate_auto_frames"]
            diff = 0.0
            for k in ref["scores"]["all"]:
                diff = max(diff, max(abs(a - b) / abs(b) for a, b in zip(ours["scores"]["all"][k], ref["scores"]["all"][k])))
            for k in ref["scores"]["mean"]:
                diff = max(diff, abs(ours["scores"]["mean"][k] - ref["scores"]["mean"][k]) / abs(ref["scores"]["mean"][k]))
            row = dict(problem=problem, grid=list(synth.grid(problem)), act_dtype=act, batch_size=bs,
                       **{f"{k}_s": stats(v) for k, v in times.items()},
                       speedup_median_dataset=float(np.median(times["loop"]) / np.median(times["evaluate_auto_dataset"])),
                       speedup_median_frames=float(np.median(times["loop"]) / np.median(times["evaluate_auto_frames"])),
                       preds_equal=bool(torch.equal(ours["preds"], ref["preds"])
                                        and torch.equal(first["evaluate_auto_dataset"]["preds"], ref["preds"])),
                       max_rel_score_diff=diff, mean_scores=ours["scores"]["mean"])
            res["configs"].append(row)
            print(json.dumps(row), flush=True)
        del frames
        torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
