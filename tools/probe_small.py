"""Small-N crossover between the strict FFMA kernel and the BF16X3 tensor-core path (what AUTO should pick)."""
import os
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs

g = _libs.load_pkg()
for N in (256, 384, 512, 640, 768, 896, 1024, 1152, 1280):
    A = torch.rand(N, N, device="cuda") - 0.5
    B = torch.rand(N, N, device="cuda") - 0.5
    C = torch.empty(N, N, device="cuda")
    row = []
    for md in (0, 2, 3, 1):
        for _ in range(5):
            g.gemm_f32(A, B, out=C, mode=md)
        best = 1e9
        for _ in range(3):
            torch.cuda.synchronize()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            for _ in range(50):
                g.gemm_f32(A, B, out=C, mode=md)
            e.record()
            torch.cuda.synchronize()
            best = min(best, s.elapsed_time(e) / 50)
        row.append(f"mode{md} {best*1e3:7.1f} us {2*N**3/best/1e9:7.1f} TF {g.last_kernel()}")
    print(f"N={N:5d} | " + " | ".join(row), flush=True)
