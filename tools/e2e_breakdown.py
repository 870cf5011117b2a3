"""Where the per-step host round trip goes: pinned H2D / D2H rates, device time per chunk size, chunked e2e."""
import os, sys, time
import torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from bench import build_model, timed_e2e, timed_rollout
from cfdbench_b200 import synth

def ev_time(fn, n=20):
    fn(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n): fn()
    b.record(); torch.cuda.synchronize()
    return a.elapsed_time(b) / n

for mb in (2, 8, 12):
    h = torch.empty(mb << 20, dtype=torch.uint8).pin_memory()
    d = torch.empty(mb << 20, dtype=torch.uint8, device="cuda")
    t1 = ev_time(lambda: d.copy_(h, non_blocking=True))
    t2 = ev_time(lambda: h.copy_(d, non_blocking=True))
    print(f"{mb} MiB pinned: H2D {t1*1e3:.0f} us ({mb*1.048576/t1:.1f} GB/s)  D2H {t2*1e3:.0f} us ({mb*1.048576/t2:.1f} GB/s)")

p = synth.n_case_params("cavity")
for b in (32, 64, 128, 256):
    batch = synth.make_batch(1, b, "cavity", with_label=False)
    inp, cp, mk = (torch.from_numpy(batch[k]).cuda() for k in ("inputs", "case_params", "mask"))
    m, _ = build_model("bf16", p)
    m.graph_rollout = False
    timed_rollout(m, inp, cp, mk, 20, 3)
    t, _ = timed_rollout(m, inp, cp, mk, 20, 3)
    m.graph_rollout = True
    timed_rollout(m, inp, cp, mk, 20, 3)
    tg, _ = timed_rollout(m, inp, cp, mk, 20, 3)
    print(f"B={b}: device step {1e6*t/20:.1f} us  (graph {1e6*tg/20:.1f} us)  -> x{256//b} = {1e6*t/20*256/b:.0f} us")
    del m
batch = synth.make_batch(1, 256, "cavity", with_label=False)
m, _ = build_model("bf16", p)
timed_e2e(m, batch, 5, 2)
t, _, _ = timed_e2e(m, batch, 20, 2)
print(f"chunked e2e: {20 / t:.1f} steps/s ({1e3 * t / 20:.3f} ms/step)")
