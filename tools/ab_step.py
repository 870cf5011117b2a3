"""Same-box A/B of the rollout step: `python tools/ab_step.py default|<tag>` times 7 x 20 graph-replayed steps (B=256, bf16)
with libcfdbench_b200.so or with a variant built into cfdbench_b200/build/<tag>/lib.so (nvcc -D... of the same sources).
Alternate the tags inside ONE process on one GPU: the step time of a power-capped card drifts between runs."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cfdbench_b200 import _lib
tag = sys.argv[1]
if tag != "default":
    _lib.LIB_PATH = os.path.join(os.path.dirname(_lib.LIB_PATH), "build", tag, "lib.so")
import numpy as np, torch, bench
from cfdbench_b200 import synth
m, _ = bench.build_model("bf16", 5)
batch = synth.make_batch(1, 256, "cavity", with_label=False)
inp, cp, mk = (torch.from_numpy(batch[k]).cuda() for k in ("inputs", "case_params", "mask"))
with torch.no_grad():
    for _ in range(3): m.generate_many(inp, cp, mk, 20)
    ts = []
    for _ in range(7):
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); m.generate_many(inp, cp, mk, 20); z.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(z) / 20)
print(f"{tag:9s}: median {np.median(ts):.4f} ms/step, min {min(ts):.4f}", flush=True)
