"""`train_auto` -- the reference's training loop (src/train_auto.py:181-313) with every step replayed from a CUDA graph
-- against that loop restated eagerly with the drop-in model: bit-identical parameters, optimizer state and losses;
the reference's output files; one synchronisation per epoch; flat peak memory; and the reference's test_multistep on
the output directory."""
import json
import os
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from test_gpu_eval_auto import _AutoSplit, _model

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SRC = os.path.join(ROOT, "oracle", "_ref", "src")


def _eager_loop(model, frames, num_epochs, lr, lr_step_size, lr_gamma, batch_size, eval_interval, generator):
    """The loop a user writes today with the drop-in pieces: DeviceFrames.loader, model(**batch), nmse.backward(),
    FusedAdam.step(), zero_grad(), .item(), a real StepLR, and the evaluation loader's RNG draw."""
    from cfdbench_b200 import FusedAdam
    from cfdbench_b200.train import dev_eval_draw
    opt = FusedAdam(model.parameters(), lr=lr)
    sched = torch.optim.lr_scheduler.StepLR(opt, step_size=lr_step_size, gamma=lr_gamma)
    losses = []
    for ep in range(num_epochs):
        for batch in frames.loader(batch_size, shuffle=True, generator=generator):
            loss = model(**batch)["loss"]
            loss["nmse"].backward()
            opt.step()
            opt.zero_grad()
            losses.append(loss["nmse"].item())
        sched.step()
        if (ep + 1) % eval_interval == 0:
            dev_eval_draw(generator)
    return losses, opt


CASES = [  # problem, act_dtype, n, batch_size, lr_step_size, lr_gamma, explicit generator
    ("cavity", "float32", 37, 8, 1, 0.5, True),
    ("cavity", "bfloat16", 24, 8, 2, 0.9, False),
    ("cylinder", "float32", 11, 1, 1, 0.9, True),
    ("tube", "float32", 21, 8, 1, 0.9, True),
    ("cavity", "float32", 5, 8, 1, 0.9, True),    # N < B: one ragged batch per epoch
]


@pytest.mark.parametrize("problem,act_dtype,n,batch_size,lr_step_size,lr_gamma,explicit", CASES)
def test_train_auto_is_bit_identical_to_the_eager_loop(tmp_path, problem, act_dtype, n, batch_size, lr_step_size,
                                                       lr_gamma, explicit):
    from cfdbench_b200 import DeviceFrames, train_auto
    epochs, eval_interval = 3, 2
    ds, dev = _AutoSplit(n, problem, seed=21), _AutoSplit(4, problem, seed=22)
    ref_m, m = _model(problem, act_dtype, seed=8), _model(problem, act_dtype, seed=8)
    frames = DeviceFrames(ds, device="cuda")
    seed = 1234
    if explicit:
        ref_losses, ref_opt = _eager_loop(ref_m, frames, epochs, 1e-3, lr_step_size, lr_gamma, batch_size, eval_interval,
                                          torch.Generator().manual_seed(seed))
        out = train_auto(m, ds, dev, tmp_path, num_epochs=epochs, lr=1e-3, lr_step_size=lr_step_size, lr_gamma=lr_gamma,
                         batch_size=batch_size, eval_batch_size=3, eval_interval=eval_interval,
                         generator=torch.Generator().manual_seed(seed))
    else:
        torch.manual_seed(seed)
        ref_losses, ref_opt = _eager_loop(ref_m, frames, epochs, 1e-3, lr_step_size, lr_gamma, batch_size, eval_interval,
                                          None)
        torch.manual_seed(seed)
        out = train_auto(m, ds, dev, tmp_path, num_epochs=epochs, lr=1e-3, lr_step_size=lr_step_size, lr_gamma=lr_gamma,
                         batch_size=batch_size, eval_batch_size=3, eval_interval=eval_interval)
    losses, opt = out["train_losses"], out["optimizer"]
    steps = -(-n // batch_size)
    assert len(losses) == len(ref_losses) == epochs * steps
    worst_p = max(float((a - b).abs().max()) for a, b in zip(m.parameters(), ref_m.parameters()))
    print(f"{problem} {act_dtype} N={n} B={batch_size}: max |param diff| {worst_p:.3e}, "
          f"max |loss diff| {max(abs(a - b) for a, b in zip(losses, ref_losses)):.3e}")
    assert losses == ref_losses
    for (name, a), b in zip(m.named_parameters(), ref_m.parameters()):
        assert torch.equal(a, b), name
        sa, sb = opt.state[a], ref_opt.state[b]
        assert torch.equal(sa["exp_avg"], sb["exp_avg"]), name
        assert torch.equal(sa["exp_avg_sq"], sb["exp_avg_sq"]), name
        assert torch.equal(sa["step"], sb["step"]) and float(sa["step"]) == epochs * steps
    assert opt.param_groups[0]["lr"] == ref_opt.param_groups[0]["lr"]
    adam = torch.optim.Adam(m.parameters(), lr=1e-3)
    adam.load_state_dict(opt.state_dict())   # the state is torch.optim.Adam's
    assert json.load(open(tmp_path / "train_losses.json")) == losses


def test_train_auto_frozen_parameters_match_the_eager_loop(tmp_path):
    """Parameters with requires_grad=False get no .grad, so FusedAdam.step neither updates them nor creates their state;
    train_auto does the same."""
    from cfdbench_b200 import DeviceFrames, train_auto
    frozen = ("fc0.weight", "blocks.1.conv0.weights2", "blocks.2.w0.bias", "fc2.bias")
    ds, dev = _AutoSplit(19, "cavity", seed=5), _AutoSplit(4, "cavity", seed=6)
    ref_m, m = _model("cavity", seed=4), _model("cavity", seed=4)
    for model in (ref_m, m):
        for name, prm in model.named_parameters():
            prm.requires_grad_(name not in frozen)
    init = {k: v.detach().clone() for k, v in m.named_parameters()}
    frames = DeviceFrames(ds, device="cuda")
    ref_losses, ref_opt = _eager_loop(ref_m, frames, 3, 1e-3, 1, 0.9, 8, 1000, torch.Generator().manual_seed(7))
    out = train_auto(m, ds, dev, tmp_path, num_epochs=3, batch_size=8, eval_interval=1000,
                     generator=torch.Generator().manual_seed(7))
    assert out["train_losses"] == ref_losses
    opt = out["optimizer"]
    for (name, a), b in zip(m.named_parameters(), ref_m.parameters()):
        assert torch.equal(a, b), name
        if name in frozen:
            assert torch.equal(a, init[name]) and a not in opt.state and b not in ref_opt.state, name
        else:
            assert not torch.equal(a, init[name]), name
            for k in ("step", "exp_avg", "exp_avg_sq"):
                assert torch.equal(opt.state[a][k], ref_opt.state[b][k]), (name, k)


def test_train_auto_output_files_and_rebuilt_caches(tmp_path):
    from cfdbench_b200 import DeviceFrames, Fno2d, evaluate_auto, train_auto
    from cfdbench_b200.loss import loss_name_to_fn
    ds, dev = _AutoSplit(20, "cavity", seed=3), _AutoSplit(7, "cavity", seed=4)
    m = _model("cavity", seed=9)
    with torch.no_grad():   # packs the weights and captures an inference graph before training
        m.generate_many(torch.randn(3, 2, 64, 64, device="cuda"), torch.randn(3, 5, device="cuda"),
                        torch.ones(3, 1, 64, 64, device="cuda"), 3)
    out = train_auto(m, ds, dev, tmp_path, num_epochs=4, batch_size=8, eval_batch_size=3, eval_interval=2, log_interval=2)
    losses = out["train_losses"]
    assert len(losses) == 4 * 3 and json.load(open(tmp_path / "train_losses.json")) == losses
    frames = DeviceFrames(dev, device="cuda")

    def fresh(sd):
        f = Fno2d(in_chan=2, out_chan=2, n_case_params=5, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
                  modes1=12, modes2=12)
        f.load_state_dict(sd)
        return f.cuda()
    for ep in (1, 3):
        ck = tmp_path / f"ckpt-{ep}"
        assert sorted(os.listdir(ck)) == ["dev_scores.json", "model.pt", "scores.json", "train_loss.json"]
        sc = json.load(open(ck / "scores.json"))
        assert list(sc) == ["ep", "train_loss", "dev_loss", "time"] and sc["ep"] == ep
        assert json.load(open(ck / "train_loss.json")) == losses[3 * ep:3 * ep + 3]
        assert sc["train_loss"] == float(np.mean(losses[3 * ep:3 * ep + 3]))
        fm = fresh(torch.load(ck / "model.pt"))
        res = evaluate_auto(fm, frames, batch_size=3)
        print(f"ckpt-{ep}: dev_loss {sc['dev_loss']!r} against {float(np.mean(res['scores']['all']['nmse']))!r}")
        assert sc["dev_loss"] == float(np.mean(res["scores"]["all"]["nmse"]))
        assert json.load(open(ck / "dev_scores.json")) == json.loads(json.dumps(res["scores"]))
        assert open(ck / "scores.json").read().startswith('{\n  "ep": ')   # dump_json's indent=2
    # the trained model's own forward / generate use the trained weights (the packed cache was rebuilt)
    fm = fresh(m.state_dict())
    x, cp = torch.randn(3, 2, 64, 64, device="cuda"), torch.randn(3, 5, device="cuda")
    mk = torch.ones(3, 1, 64, 64, device="cuda")
    with torch.no_grad():
        a, b = m.generate(x, cp, mk), fm.generate(x, cp, mk)
        a2, b2 = m.generate_many(x, cp, mk, 3)[-1], fm.generate_many(x, cp, mk, 3)[-1]
    assert torch.equal(a, b) and torch.equal(a2, b2)
    final = fresh(torch.load(tmp_path / "ckpt-3" / "model.pt"))
    with torch.no_grad():
        assert torch.equal(final.generate(x, cp, mk), a)
    # a second run into the same directory backs the previous checkpoint up, as the reference does
    prev = open(tmp_path / "ckpt-1" / "model.pt", "rb").read()
    train_auto(m, ds, dev, tmp_path, num_epochs=2, batch_size=8, eval_batch_size=3, eval_interval=2)
    assert open(tmp_path / "ckpt-1" / "backup_model.pt", "rb").read() == prev


def _count_syncs(fn):
    torch.cuda.synchronize()
    prev = torch.cuda.get_sync_debug_mode()
    with warnings.catch_warnings(record=True) as caught:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode(prev)
    return [str(w.message) for w in caught if "called a synchronizing CUDA operation" in str(w.message)]


def test_train_auto_syncs_and_memory(tmp_path):
    from cfdbench_b200 import DeviceFrames, train_auto
    m = _model("cavity", seed=6)
    dev = DeviceFrames(_AutoSplit(4, "cavity", seed=1), device="cuda")
    splits = {n: DeviceFrames(_AutoSplit(n, "cavity", seed=2), device="cuda") for n in (32, 37, 40, 128)}

    def run(n, epochs):
        return train_auto(m, splits[n], dev, tmp_path, num_epochs=epochs, batch_size=8, eval_interval=1000)
    run(32, 1)   # warms the model's workspace and packed-weight tables
    counts = {}
    for epochs in (1, 3):
        syncs = _count_syncs(lambda: run(32, epochs))
        print(f"{epochs} epochs: {len(syncs)} synchronising operations", syncs[:3])
        counts[epochs] = len(syncs)
    assert counts == {1: 1, 3: 3}

    def rise(n, epochs):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        run(n, epochs)
        torch.cuda.synchronize()
        return torch.cuda.max_memory_allocated() - base
    r2, r6 = rise(32, 2), rise(32, 6)
    r_small, r_large = rise(32, 2), rise(128, 2)
    r_even, r_ragged = rise(40, 2), rise(37, 2)
    print(f"peak rise: 2 epochs {r2} B, 6 epochs {r6} B; N=32 {r_small} B, N=128 {r_large} B; "
          f"N=40 {r_even} B, N=37 (ragged) {r_ragged} B")
    assert r6 <= r2 + 4096
    # what grows with N: the permutation (8 B per sample), the coefficient table and log (28 B per step), rounding
    assert r_large - r_small <= 8 * 96 + 28 * 12 + 8192
    assert r_ragged <= r_even + 2 * 2 ** 20


class _Learnable(_AutoSplit):
    """label = a fixed smooth map of the input: a task the network can fit."""

    def __init__(self, n, seed=0):
        super().__init__(n, "cavity", seed=seed)
        rng = np.random.default_rng(seed)
        h = np.linspace(0, 2 * np.pi, 64, dtype=np.float32)
        fields = np.zeros((n, 2, 64, 64), np.float32)
        for k in range(1, 4):
            a = rng.standard_normal((n, 2, 1, 1)).astype(np.float32) / k
            fields += a * np.sin(k * h)[None, None, :, None] * np.cos(k * h)[None, None, None, :]
        self.inputs[:, :2] = torch.from_numpy(fields)
        self.inputs[:, 2] = 1.0
        self.labels[:, :2] = torch.from_numpy(0.8 * fields)
        self.labels[:, 2] = 1.0


def test_train_auto_learns(tmp_path):
    from cfdbench_b200 import train_auto
    m = _model("cavity", seed=2)
    out = train_auto(m, _Learnable(64, seed=1), _Learnable(8, seed=2), tmp_path, num_epochs=6, batch_size=8,
                     eval_interval=1000, generator=torch.Generator().manual_seed(0))
    per_epoch = np.asarray(out["train_losses"]).reshape(6, 8).mean(axis=1)
    print("mean nmse per epoch:", per_epoch)
    assert np.all(np.isfinite(per_epoch)) and per_epoch[-1] < 0.5 * per_epoch[0]


_REF_TRAIN = r"""
import sys
sys.path.insert(0, {root!r})
from cfdbench_b200 import runner
runner.install({src!r}, stub_missing=True)
sys.argv = ["train_auto.py"] + {argv!r}
from args import Args
from dataset import get_auto_dataset
from utils.common import get_output_dir
from utils.autoregressive import init_model
from pathlib import Path
from cfdbench_b200 import train_auto
args = Args().parse_args()
out = get_output_dir(args, is_auto=True)
train_data, dev_data, _ = get_auto_dataset(data_dir=Path(args.data_dir), data_name=args.data_name,
                                           delta_time=args.delta_time, norm_props=bool(args.norm_props),
                                           norm_bc=bool(args.norm_bc))
model = init_model(args)
train_auto(model, train_data, dev_data, out, num_epochs=2, lr=args.lr, batch_size=4, eval_batch_size=2, eval_interval=1,
           log_interval=2)
print("TRAINED", out)
"""


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF_SRC, "models", "fno")),
                    reason="oracle/_ref/src (installed by __graft_entry__.build()) is not present")
def test_reference_test_multistep_reads_train_auto_output(tmp_path):
    from test_gpu_runner import COMMON, run_script
    import shutil
    src = str(tmp_path / "src")
    shutil.copytree(REF_SRC, src)
    for root, dirs, files in os.walk(src):
        os.chmod(root, 0o755)
        for f in files:
            os.chmod(os.path.join(root, f), 0o644)
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import make_tiny_cavity
    data = str(tmp_path / "data")
    os.makedirs(data)
    make_tiny_cavity.make(data)
    out = str(tmp_path / "result")
    argv = COMMON + ["--data_dir", data, "--output_dir", out]
    env = {**os.environ, "PYTHONPATH": ROOT + os.pathsep + os.environ.get("PYTHONPATH", ""), "PYTHONDONTWRITEBYTECODE": "1"}
    r = subprocess.run([sys.executable, "-c", _REF_TRAIN.format(root=ROOT, src=src, argv=argv)], capture_output=True,
                       text=True, env=env, cwd=src, timeout=600)
    assert r.returncode == 0, (r.stdout[-1500:], r.stderr[-3000:])
    run_dir = os.path.join(out, "auto", "cavity_prop_bc_geo", "dt0.1", "fno", "lr0.001_d4_h32_m112_m212")
    assert os.path.isfile(os.path.join(run_dir, "ckpt-1", "scores.json")), os.listdir(out)
    r3 = run_script(src, "test_multistep.py", data, out, [])
    assert r3.returncode == 0, (r3.stdout[-1500:], r3.stderr[-3000:])
    metrics = json.load(open(os.path.join(run_dir, "multistep_metrics.json")))
    assert len(metrics) == 20 and all(np.isfinite(x["nmse"]) for x in metrics)
