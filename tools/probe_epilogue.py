"""What the fused bias / activation epilogue costs, and what it saves (b200_gemm_bf16_epi / b200_gemm_f16_epi).

Shapes: 4096^3 and 8192^3 (NN) and an MLP up-projection x @ W.t() with m = 8192, n = 16384, k = 4096 (NT: W is
stored n x k, as nn.Linear holds it).  bf16 and fp16 operands, 16-bit C.  Variants, alternating inside each round so
that drift of the shared card hits them alike:
  plain          the _ex call, (alpha, beta) = (1, 0): the plain kernel
  bias           bias vector, B200_ACT_NONE
  bias+relu, bias+gelu, bias+gelu_tanh
  unfused        the plain GEMM, then torch's C.add_(bias) and F.gelu(C): what a caller does without the epilogue
GEMM kernel time comes from b200_gemm_debug_kernel_timing; whole-call time from CUDA events around a batch of calls
(the unfused baseline is timed this way only, against bias+gelu).  Each figure is the median over rounds.  Prints the
card name, power limit and maximum SM clock from the same run, one line per (shape, type, variant), and writes the
table as JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs

SHAPES = {"4096^3 NN": (4096, 4096, 4096, 0), "8192^3 NN": (8192, 8192, 8192, 0), "MLP NT": (8192, 16384, 4096, 1)}
ACT = {"plain": None, "bias": 0, "bias+relu": 1, "bias+gelu": 2, "bias+gelu_tanh": 3}
VARIANTS = list(ACT) + ["unfused"]


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
    ap.add_argument("--shapes", default=",".join(SHAPES))
    ap.add_argument("--types", default="bf16,f16")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    g = _libs.load_pkg()
    lib = g.lib
    info = card()
    print("card:", info, flush=True)
    rows = []
    for shape in args.shapes.split(","):
        m, n, k, op_b = SHAPES[shape]
        for ty in args.types.split(","):
            d, ot = (torch.bfloat16, 1) if ty == "bf16" else (torch.float16, 2)
            ex, epi = (lib.b200_gemm_bf16_ex, lib.b200_gemm_bf16_epi) if ty == "bf16" else (lib.b200_gemm_f16_ex, lib.b200_gemm_f16_epi)
            gen = torch.Generator(device="cuda").manual_seed(m + n + k)
            A = (torch.rand((m, k), device="cuda", generator=gen) * 2 - 1).to(d)
            B = (torch.rand((n, k) if op_b else (k, n), device="cuda", generator=gen) * 2 - 1).to(d)
            bias = (torch.rand(n, device="cuda", generator=gen) * 2 - 1).to(d)
            Cb = torch.empty((m, n), device="cuda", dtype=d)
            ldb = k if op_b else n
            st = torch.cuda.current_stream().cuda_stream

            def call(v):
                if v == "unfused":
                    assert ex(0, op_b, m, n, k, 1.0, A.data_ptr(), k, B.data_ptr(), ldb, 0.0, Cb.data_ptr(), n, ot, st) == 0
                    Cb.add_(bias)
                    F.gelu(Cb)
                elif ACT[v] is None:
                    assert ex(0, op_b, m, n, k, 1.0, A.data_ptr(), k, B.data_ptr(), ldb, 0.0, Cb.data_ptr(), n, ot, st) == 0
                else:
                    assert epi(0, op_b, m, n, k, 1.0, A.data_ptr(), k, B.data_ptr(), ldb, 0.0, Cb.data_ptr(), n, ot,
                               bias.data_ptr(), ACT[v], st) == 0

            iters = max(2, int(1e13 / (2.0 * m * n * k)))
            calls, kern, names = {v: [] for v in VARIANTS}, {v: [] for v in VARIANTS}, {}
            for v in VARIANTS:                                 # warm every variant (maps, modules)
                for _ in range(2):
                    call(v)
                names[v] = g.last_kernel()
            torch.cuda.synchronize()
            for _ in range(args.rounds):
                for v in VARIANTS:
                    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    lib.b200_gemm_debug_kernel_timing(1)
                    s.record()
                    for _ in range(iters):
                        call(v)
                    e.record()
                    torch.cuda.synchronize()
                    ksum, cnt = g.kernel_time_ms()
                    lib.b200_gemm_debug_kernel_timing(0)
                    calls[v].append(s.elapsed_time(e) / iters)
                    kern[v].append(ksum / max(cnt, 1))
            med = {v: (statistics.median(calls[v]), statistics.median(kern[v])) for v in VARIANTS}
            flop = 2.0 * m * n * k
            for v in VARIANTS:
                c, kt = med[v]
                row = dict(shape=shape, m=m, n=n, k=k, type=ty, variant=v, kernel_name=names[v], call_ms=c, kernel_ms=kt,
                           kernel_tflops=flop / kt / 1e9, spread_kernel_ms=[min(kern[v]), max(kern[v])],
                           spread_call_ms=[min(calls[v]), max(calls[v])])
                extra = ""
                if v != "plain":
                    row["kernel_cost_vs_plain"] = kt / med["plain"][1] - 1.0
                    row["call_cost_vs_plain"] = c / med["plain"][0] - 1.0
                    extra += f"  vs plain: kernel {100 * row['kernel_cost_vs_plain']:+.1f} %  call {100 * row['call_cost_vs_plain']:+.1f} %"
                if v == "unfused":
                    row["fused_saves"] = 1.0 - med["bias+gelu"][0] / c
                    extra += f"  fused bias+gelu saves {100 * row['fused_saves']:.1f} % of the call"
                rows.append(row)
                print(f"{shape:10s} {ty:4s} {v:15s} call {c:7.3f} ms  kernel {kt:7.3f} ms {row['kernel_tflops']:6.1f} TFLOP/s"
                      f"{extra}  {names[v]}", flush=True)
            del A, B, Cb
            torch.cuda.empty_cache()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
