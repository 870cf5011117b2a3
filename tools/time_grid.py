"""Timing of the grid-generic fp32 path on this GPU.  The card name and power limit are read in the same run.

At batch `--batch` (default 256), fp32 storage, CUDA events, median of `--reps` repetitions:
  * the 20-step device rollout (generate_many on device tensors, graph-replayed) per step, and
  * the training step (forward + nmse.backward() + FusedAdam.step()),
for 66x65 on the grid path, 64x64 on the grid path (generic_grid_at_64), 64x64 on the 64x64 fp32 kernels, and the
reference Fno2d with torch defaults on the same GPU (oracle/_ref when build() installed it, else the torch port);
then CUDA-event times of every grid kernel at 66x65 and their algorithmic bytes (32*H*W*4 read + write per sample-layer)
over kernel time.

    python tools/time_grid.py [--batch 256] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main() -> None:
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import ctypes as C
    import numpy as np
    import torch
    from cfdbench_b200 import Fno2d, _lib, loss_name_to_fn, synth
    from cfdbench_b200.optim import FusedAdam

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    try:
        power = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader"],
                               capture_output=True, text=True, timeout=60).stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    gpu = torch.cuda.get_device_name(dev)
    B, S = args.batch, args.steps
    print(f"# {gpu}, power limit {power}; B={B}, fp32 storage, median of {args.reps}", flush=True)
    rec = dict(gpu=gpu, power_limit=power, batch=B, rollout_steps=S, results={}, kernels_66x65={})

    def timed(fn, warm=2):
        for _ in range(warm):
            fn()
        ts = []
        for _ in range(args.reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fn()
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        return float(np.median(ts))

    sd = synth.make_state_dict(0, n_params=5, spectral_gain=50.0)

    def data(problem):
        bt = synth.make_batch(1, B, problem)
        return {k: torch.from_numpy(v).to(dev) for k, v in bt.items()}

    def ours(tb, generic):
        m = Fno2d(in_chan=2, out_chan=2, n_case_params=5, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
                  modes1=12, modes2=12)
        m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
        m.generic_grid_at_64 = generic
        opt = FusedAdam(m.parameters(), lr=1e-4)

        def roll():
            with torch.no_grad():
                m.generate_many(tb["inputs"], tb["case_params"], tb["mask"], S)

        def train():
            opt.zero_grad(set_to_none=True)
            m(**tb)["loss"]["nmse"].backward()
            opt.step()
        return roll, train

    def reference(tb):
        ref_src = os.path.join(ROOT, "oracle", "_ref", "src")
        if os.path.isdir(os.path.join(ref_src, "models", "fno")):
            sys.path.insert(0, ref_src)
            from models.fno.fno2d import Fno2d as Ref
            from models.loss import loss_name_to_fn as ref_loss
            m = Ref(in_chan=2, out_chan=2, n_case_params=5, loss_fn=ref_loss("nmse"), num_layers=4, hidden_dim=32,
                    modes1=12, modes2=12)
            m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
            m = m.to(dev)
            label = "reference Fno2d (oracle/_ref), torch defaults"

            def fwd(**kw):
                return m(**kw)

            def many(x, cp, mk, n):
                return m.generate_many(x, cp, mk, n)
            params = list(m.parameters())
        else:
            from oracle import fno_torch_port as port
            pp = {k: v.to(dev).requires_grad_(True) for k, v in port.params_from_numpy(sd).items()}
            label = "torch port of the reference (oracle/fno_torch_port.py), torch defaults"

            def fwd(**kw):
                return port.forward(pp, kw["inputs"], kw["case_params"], kw["mask"], kw["label"])

            def many(x, cp, mk, n):
                return port.rollout(pp, x, cp, mk, n)
            params = list(pp.values())
        opt = torch.optim.Adam(params, lr=1e-4)

        def roll():
            with torch.no_grad():
                many(tb["inputs"], tb["case_params"], tb["mask"], S)

        def train():
            opt.zero_grad(set_to_none=True)
            fwd(**tb)["loss"]["nmse"].backward()
            opt.step()
        return label, roll, train

    tube, cav = data("tube"), data("cavity")
    cases = [("66x65 grid path", tube, True, 66 * 65), ("64x64 grid path", cav, True, 64 * 64),
             ("64x64 fp32 fast path", cav, False, 64 * 64)]
    for name, tb, generic, pix in cases:
        roll, train = ours(tb, generic)
        r = timed(roll) / S
        t = timed(train)
        rec["results"][name] = dict(rollout_ms_per_step=r, train_step_ms=t, rollout_ns_per_sample_pixel=r * 1e6 / (B * pix),
                                    train_ns_per_sample_pixel=t * 1e6 / (B * pix))
        print(f"{name:28s} rollout {r:8.3f} ms/step   train step {t:8.3f} ms", flush=True)
    label, roll, train = reference(tube)
    r, t = timed(roll, warm=1) / S, timed(train, warm=1)
    rec["results"]["66x65 " + label] = dict(rollout_ms_per_step=r, train_step_ms=t)
    print(f"66x65 {label}: rollout {r:8.3f} ms/step   train step {t:8.3f} ms", flush=True)

    # per-kernel CUDA-event times at 66x65 through the ABI
    lib, gh, gw = _lib.load(), 66, 65
    m = Fno2d(in_chan=2, out_chan=2, n_case_params=5, loss_fn=loss_name_to_fn("nmse"), num_layers=4, hidden_dim=32,
              modes1=12, modes2=12)
    m.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    pk = m._pack(need_bwd=True)
    w = m._coords(pk, gh, gw)[0]
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    a0, a1, pre = (torch.randn(B, 32, gh, gw, device=dev) for _ in range(3))
    xm = torch.empty(288, B, 32, dtype=torch.complex64, device=dev)
    ym = torch.randn(288, B, 32, dtype=torch.complex64, device=dev)
    z = torch.empty(B, gh, 24, 32, device=dev)
    preds = torch.empty(B, 2, gh, gw, device=dev)
    dpre = torch.empty(B, 32, gh, gw, device=dev)
    dz1 = torch.empty(min(B, _lib.BWD_CHUNK), 128, gh, gw, device=dev)
    part = torch.empty(lib.fno_grid_bwd_partials_bytes(gh, gw), dtype=torch.uint8, device=dev)
    gr = [torch.empty(n, device=dev) for n in (4096, 128, 256, 2)]
    w0t, b0 = pk["w0t"][0], m.blocks[0].w0.bias
    inv = 1.0 / (gh * gw)
    plane_bytes = 32 * gh * gw * 4 * 2 * B   # one hidden tensor read + one written, per layer
    kern = {
        "lift": lambda: lib.fno_grid_lift_fwd(tube["inputs"].data_ptr(), tube["mask"].data_ptr(), tube["case_params"].data_ptr(),
                                              C.byref(w), a0.data_ptr(), B, gh, gw, st),
        "dft_fwd": lambda: lib.fno_grid_spectral_dft_fwd(a0.data_ptr(), xm.data_ptr(), B, gh, gw, 1.0, 1.0, st),
        "mode_mix (shared)": lambda: lib.fno_mode_mix(xm.data_ptr(), pk["struct"].spec_wk[0], ym.data_ptr(), B, st),
        "inv_kx": lambda: lib.fno_grid_spectral_inv_kx(ym.data_ptr(), z.data_ptr(), B, gh, gw, inv, 2 * inv, st),
        "block_out GELU_SAVE_PRE": lambda: lib.fno_grid_block_out(1, z.data_ptr(), a0.data_ptr(), w0t.data_ptr(), b0.data_ptr(),
                                                                  a1.data_ptr(), pre.data_ptr(), None, B, gh, gw, st),
        "block_out GELU": lambda: lib.fno_grid_block_out(0, z.data_ptr(), a0.data_ptr(), w0t.data_ptr(), b0.data_ptr(),
                                                         a1.data_ptr(), None, None, B, gh, gw, st),
        "project": lambda: lib.fno_grid_project_fwd(a1.data_ptr(), tube["mask"].data_ptr(), C.byref(w), preds.data_ptr(), B,
                                                    gh, gw, st),
        "project_bwd + fc1/fc2 grads": lambda: lib.fno_grid_project_bwd(a1.data_ptr(), preds.data_ptr(), tube["mask"].data_ptr(),
                                                                        pre.data_ptr(), C.byref(w), dpre.data_ptr(),
                                                                        dz1.data_ptr(), part.data_ptr(),
                                                                        *[t.data_ptr() for t in gr], B, gh, gw, st),
    }
    for name, fn in kern.items():
        def call(fn=fn, name=name):
            _lib.check(fn(), name)
        ms = timed(call)
        rec["kernels_66x65"][name] = dict(ms=ms, algorithmic_GBps=plane_bytes / (ms * 1e-3) / 1e9)
        print(f"  {name:30s} {ms * 1e3:9.1f} us   {plane_bytes / (ms * 1e-3) / 1e9:7.1f} GB/s (32*H*W*4*2 per sample)",
              flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rec, f, indent=1)


if __name__ == "__main__":
    main()
