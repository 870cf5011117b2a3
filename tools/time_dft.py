"""Standalone timing of fno_spectral_dft_fwd at B=256 (bf16 planes: dft_fwd_tc_kernel, fp32 planes: dft_fwd_kernel):
median of 30 event-bracketed launches, L2 flushed between launches by the 67 MB / 134 MB input itself being larger
than what survives."""
import ctypes as C, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from cfdbench_b200 import _lib
lib = _lib.load()
b = 256
st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
for name, dt, code in (("bf16", torch.bfloat16, _lib.ACT_BF16), ("f32", torch.float32, _lib.ACT_F32)):
    x = torch.randn(b, 32, 64, 64, device="cuda").to(dt)
    x2 = torch.randn(b, 32, 64, 64, device="cuda").to(dt)
    xm = torch.empty(288, b, 32, dtype=torch.complex64, device="cuda")
    ts = []
    for i in range(34):
        src = x if i % 2 == 0 else x2
        a, z = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        _lib.check(lib.fno_spectral_dft_fwd(src.data_ptr(), xm.data_ptr(), b, code, 1.0, 1.0, st), "dft")
        z.record()
        torch.cuda.synchronize()
        if i >= 4:
            ts.append(a.elapsed_time(z) * 1e3)
    print(f"dft_fwd {name}: median {np.median(ts):.1f} us, min {min(ts):.1f} us")
