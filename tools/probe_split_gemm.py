"""Split-precision fp32 GEMM kernels at N^3 (b200_gemm_f32 in F16X2, BF16X3 and BF16X2 mode), the tree it is run from.

Per mode and size: the GEMM kernel's own time (b200_gemm_debug_kernel_timing: CUDA events around each launch) and the
whole call's (events around a batch of calls, pre-pass included), each the median over rounds in which every mode
alternates, and a SHA-256 of C for seeded operands, so that two builds run one after the other can be compared for
speed and for C bit for bit.  Prints the card's name, power limit and maximum SM clock, one line per (N, mode), and
writes the table as JSON to the file named by --out."""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except OSError:
        pass
    return torch.cuda.get_device_name(0) + " (power limit not readable)"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="4096,8192")
    ap.add_argument("--modes", default="F16X2,BF16X3,BF16X2")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    g = _libs.load_pkg()
    info = card()
    print("card:", info, flush=True)
    modes = {m: getattr(g, "F32_" + m) for m in args.modes.split(",")}
    rows = []
    for n in [int(x) for x in args.sizes.split(",")]:
        gen = torch.Generator(device="cuda").manual_seed(n)
        A = torch.rand((n, n), device="cuda", generator=gen) * 2 - 1
        B = torch.rand((n, n), device="cuda", generator=gen) * 2 - 1
        C = torch.empty((n, n), device="cuda")
        iters = max(2, int(2e13 / (2.0 * n ** 3)))
        names, digest = {}, {}
        for m, md in modes.items():                          # warm each mode, and hash its C
            for _ in range(2):
                g.gemm_f32(A, B, out=C, mode=md)
            torch.cuda.synchronize()
            names[m] = g.last_kernel()
            digest[m] = hashlib.sha256(C.cpu().numpy().tobytes()).hexdigest()
        calls, kern = {m: [] for m in modes}, {m: [] for m in modes}
        for _ in range(args.rounds):
            for m, md in modes.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                g.lib.b200_gemm_debug_kernel_timing(1)
                s.record()
                for _ in range(iters):
                    g.gemm_f32(A, B, out=C, mode=md)
                e.record()
                torch.cuda.synchronize()
                ksum, cnt = g.kernel_time_ms()
                g.lib.b200_gemm_debug_kernel_timing(0)
                calls[m].append(s.elapsed_time(e) / iters)
                kern[m].append(ksum / max(cnt, 1))
        for m in modes:
            c, k = statistics.median(calls[m]), statistics.median(kern[m])
            row = dict(n=n, mode=m, kernel_name=names[m], call_ms=c, kernel_ms=k, kernel_tflops=2.0 * n ** 3 / k / 1e9,
                       spread_kernel_ms=[min(kern[m]), max(kern[m])], c_sha256=digest[m])
            rows.append(row)
            print(f"N={n:5d} {m:7s} call {c:7.3f} ms  kernel {k:7.3f} ms [{min(kern[m]):.3f} .. {max(kern[m]):.3f}] "
                  f"{row['kernel_tflops']:6.1f} TFLOP/s  {names[m]}  C sha256 {digest[m][:16]}", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
