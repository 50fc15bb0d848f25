"""NN, NT, TN and TT at N^3 for bf16 -> f32, TF32, F16X2, int8 and STRICT (b200_gemm_*_op).

Per call: whole-call time (CUDA events around a batch of calls, pre-passes and transposes included) and GEMM kernel
time (b200_gemm_debug_kernel_timing: events around the wgmma / FFMA kernel only).  The four layouts alternate inside
every round, so drift of the shared card hits them alike; each figure is the median over rounds.  Prints the card
name and power limit, one line per (N, path, layout), and writes the table as JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs

LAYOUTS = {"NN": (0, 0), "NT": (0, 1), "TN": (1, 0), "TT": (1, 1)}
PATHS = ("bf16", "tf32", "f16x2", "int8", "strict")


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
    ap.add_argument("--paths", default=",".join(PATHS))
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    g = _libs.load_pkg()
    lib = g.lib
    info = card()
    print("card:", info, flush=True)
    rows = []
    for n in [int(x) for x in args.sizes.split(",")]:
        gen = torch.Generator(device="cuda").manual_seed(n)
        X = torch.rand((n, n), device="cuda", generator=gen) * 2 - 1
        Y = torch.rand((n, n), device="cuda", generator=gen) * 2 - 1
        for path in args.paths.split(","):
            if path == "bf16":
                A, B, C = X.bfloat16(), Y.bfloat16(), torch.empty((n, n), device="cuda")
                fn = lambda oa, ob: lib.b200_gemm_bf16_op(oa, ob, n, n, n, A.data_ptr(), n, B.data_ptr(), n, C.data_ptr(), n, 0, None)
            elif path == "int8":
                A = torch.randint(-127, 128, (n, n), device="cuda", generator=gen, dtype=torch.int8)
                B = torch.randint(-127, 128, (n, n), device="cuda", generator=gen, dtype=torch.int8)
                C = torch.empty((n, n), dtype=torch.int32, device="cuda")
                fn = lambda oa, ob: lib.b200_gemm_s8s32_op(oa, ob, n, n, n, A.data_ptr(), n, B.data_ptr(), n, C.data_ptr(), n, None)
            else:
                mode = {"tf32": g.F32_TF32, "f16x2": g.F32_F16X2, "strict": g.F32_STRICT}[path]
                A, B, C = X, Y, torch.empty((n, n), device="cuda")
                fn = lambda oa, ob, mode=mode: lib.b200_gemm_f32_op(oa, ob, n, n, n, 1.0, A.data_ptr(), n, B.data_ptr(), n, 0.0,
                                                                    C.data_ptr(), n, mode, None)
            iters = max(2, int(2e12 / (2.0 * n ** 3) * (0.05 if path == "strict" else 1.0)))
            calls, kern, names = {k: [] for k in LAYOUTS}, {k: [] for k in LAYOUTS}, {}
            for lay, (oa, ob) in LAYOUTS.items():                      # warm every layout (workspace, maps, modules)
                for _ in range(2):
                    assert fn(oa, ob) == 0
                names[lay] = g.last_kernel()
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for lay, (oa, ob) in LAYOUTS.items():
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    lib.b200_gemm_debug_kernel_timing(1)
                    s.record()
                    for _ in range(iters):
                        fn(oa, ob)
                    e.record()
                    torch.cuda.synchronize()
                    ksum, cnt = g.kernel_time_ms()
                    lib.b200_gemm_debug_kernel_timing(0)
                    calls[lay].append(s.elapsed_time(e) / iters)
                    kern[lay].append(ksum / max(cnt, 1))
            nn_call, nn_kern = statistics.median(calls["NN"]), statistics.median(kern["NN"])
            for lay in LAYOUTS:
                c, k = statistics.median(calls[lay]), statistics.median(kern[lay])
                flop = 2.0 * n ** 3
                row = dict(n=n, path=path, layout=lay, kernel_name=names[lay], call_ms=c, kernel_ms=k,
                           call_tflops=flop / c / 1e9, kernel_tflops=flop / k / 1e9, call_vs_nn=nn_call / c,
                           kernel_vs_nn=nn_kern / k, spread_call_ms=[min(calls[lay]), max(calls[lay])])
                rows.append(row)
                print(f"N={n:5d} {path:6s} {lay}  call {c:8.3f} ms {row['call_tflops']:6.1f} TFLOP/s ({row['call_vs_nn']:.3f} x NN)"
                      f"  kernel {k:8.3f} ms {row['kernel_tflops']:6.1f} TFLOP/s ({row['kernel_vs_nn']:.3f} x NN)  {names[lay]}",
                      flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
