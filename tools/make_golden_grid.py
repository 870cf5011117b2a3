"""TEST INFRASTRUCTURE -- generate the non-64x64 golden fixtures (tests/golden/grid/*.npz) from the UNMODIFIED reference.

Same procedure and checks as oracle/make_golden.py, for grids other than 64x64 (CFDBench's tube and dam frames are
(64 + 2) x (64 + 1) = 66x65, reference src/utils/autoregressive.py:24-26).  The fixtures live in a subdirectory because
the 64x64 suites enumerate tests/golden/*.npz.  Needs the reference tree that oracle/install_reference.py places in
the git-ignored oracle/_ref/src:

    PYTHONDONTWRITEBYTECODE=1 python tools/make_golden_grid.py [--out DIR]

For each case it builds the reference `Fno2d` with the seeded weights of `cfdbench_b200.synth`, runs forward / loss /
backward / generate_many on CPU fp32, asserts that the torch port is bit-identical and the float64 numpy oracle agrees
to <2e-6 (preds, activations, spectral output) / <5e-5 (gradients), and stores seeds + reference outputs.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True

from oracle.make_golden import ref_model  # noqa: E402  (imports the reference from oracle/_ref/src)

from cfdbench_b200 import synth  # noqa: E402
from oracle import fno_numpy as onp  # noqa: E402
from oracle import fno_torch_port as opt  # noqa: E402

CASES = [
    # name, problem, batch, weight seed, batch seed, spectral gain, rollout steps
    ("tube_b2_66x65", "tube", 2, 104, 204, 200.0, 3),
]


def make_case(problem: str, b: int, wseed: int, bseed: int, gain: float, steps: int) -> dict:
    p = synth.n_case_params(problem)
    sd = synth.make_state_dict(wseed, n_params=p, spectral_gain=gain)
    batch = synth.make_batch(bseed, b, problem)
    tb = {k: torch.from_numpy(v) for k, v in batch.items()}
    model = ref_model(sd, p)

    acts = []   # lift output and every block output
    hooks = [model.fc0.register_forward_hook(lambda m, i, o: acts.append(o.detach().numpy().copy()))]
    for blk in model.blocks:
        hooks.append(blk.register_forward_hook(lambda m, i, o: acts.append(o.detach().numpy().copy())))
    out = model(**tb)
    for hk in hooks:
        hk.remove()
    out["loss"]["nmse"].backward()
    grads = {k: v.grad.numpy().copy() for k, v in model.named_parameters()}
    with torch.no_grad():
        roll = model.generate_many(tb["inputs"], tb["case_params"], tb["mask"], steps)
        spec = model.blocks[0].conv0(torch.from_numpy(acts[0])).numpy()

    # --- pin the oracles against the reference
    pp = opt.params_from_numpy(sd, requires_grad=True)
    pout = opt.forward(pp, tb["inputs"], tb["case_params"], tb["mask"], tb["label"], return_acts=True)
    assert torch.equal(pout["preds"], out["preds"]), "torch port is not bit-identical to the reference"
    for k in out["loss"]:
        assert torch.equal(pout["loss"][k], out["loss"][k]), k
    pout["loss"]["nmse"].backward()
    for k, g in grads.items():
        assert np.array_equal(pp[k].grad.numpy(), g), f"port grad {k}"
    proll = opt.rollout(opt.params_from_numpy(sd), tb["inputs"], tb["case_params"], tb["mask"], steps)
    for a, r in zip(proll, roll):
        assert torch.equal(a, r)
    nout = onp.fno_forward(sd, batch["inputs"], batch["case_params"], batch["mask"], batch["label"], return_acts=True)
    e = onp.rel_l2(out["preds"].detach().numpy(), nout["preds"])
    assert e < 2e-6, f"numpy oracle vs reference preds rel-L2 {e}"
    for i, a in enumerate(acts):
        ea = onp.rel_l2(a, nout["acts"][i])
        assert ea < 2e-6, (i, ea)
    ngr = onp.fno_backward(sd, batch["inputs"], batch["case_params"], batch["mask"], batch["label"])
    worst = 0.0
    for k, g in grads.items():
        eg = np.linalg.norm(g - ngr[k]) / np.linalg.norm(ngr[k])
        worst = max(worst, eg)
        assert eg < 5e-5, f"numpy oracle grad {k}: {eg}"
    es = onp.rel_l2(spec, onp.spectral_conv(acts[0], sd["blocks.0.conv0.weights1"], sd["blocks.0.conv0.weights2"]))
    assert es < 2e-6, es
    print(f"numpy-vs-ref preds {e:.2e}, spectral {es:.2e}, worst grad {worst:.2e}; port bit-exact")

    store = dict(
        problem=np.array(problem), weight_seed=np.array(wseed), batch_seed=np.array(bseed),
        spectral_gain=np.array(gain), steps=np.array(steps),
        preds=out["preds"].detach().numpy(),
        loss=np.array([out["loss"][k].item() for k in ("mse", "rmse", "mae", "nmse")], dtype=np.float64),
        rollout=np.stack([r.numpy() for r in roll]),
        # hidden tensors of sample 0 on every 8th channel (0, 8, 16, 24): keeps the fixture below 1 MB
        act0_b0=acts[0][:1, ::8], act1_b0=acts[1][:1, ::8], act4_b0=acts[-1][:1, ::8],
        spectral0_b0=spec[:1, ::8],
    )
    for k in ("fc0.weight", "fc0.bias", "fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias",
              "blocks.0.w0.weight", "blocks.0.w0.bias", "blocks.3.w0.weight", "blocks.3.w0.bias"):
        store["grad::" + k] = grads[k]
    for k in ("blocks.0.conv0.weights1", "blocks.0.conv0.weights2", "blocks.3.conv0.weights1", "blocks.3.conv0.weights2"):
        store["gradslice::" + k] = grads[k][:, :, ::4, ::4]           # (32,32,3,3) complex
        store["gradnorm::" + k] = np.array(np.linalg.norm(grads[k]))
    return store


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=os.path.join(ROOT, "tests", "golden", "grid"))
    args = ap.parse_args()
    torch.set_num_threads(8)
    os.makedirs(args.out, exist_ok=True)
    for name, problem, b, wseed, bseed, gain, steps in CASES:
        store = make_case(problem, b, wseed, bseed, gain, steps)
        np.savez_compressed(os.path.join(args.out, name + ".npz"), **store)
        print(name, "written to", args.out)


if __name__ == "__main__":
    main()
