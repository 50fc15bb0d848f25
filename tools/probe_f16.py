"""fp16 against bf16 on the tensor cores at N^3, every layout (b200_gemm_f16_ex / b200_gemm_bf16_ex).

Variants per layout: bf16 -> fp32, fp16 -> fp32, bf16 -> bf16, fp16 -> fp16, and the two 16-bit-C ones again with
beta != 0 (alpha = 1, beta = 0.5: the epilogue reads C once).  Per call: whole-call time (CUDA events around a
batch of calls) and GEMM kernel time (b200_gemm_debug_kernel_timing).  Every variant of every layout alternates
inside each round, so drift of the shared card hits them alike; each figure is the median over rounds.  Prints the
card name and power limit, one line per (N, layout, variant) with the fp16 : bf16 ratio of its C class and the cost
of beta != 0, and writes the table as JSON to the file named by --out."""
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
# name: (operand type, out_type, beta)
VARIANTS = {"bf16->f32": ("bf16", 0, 0.0), "f16->f32": ("f16", 0, 0.0), "bf16->bf16": ("bf16", 1, 0.0),
            "f16->f16": ("f16", 2, 0.0), "bf16->bf16 beta": ("bf16", 1, 0.5), "f16->f16 beta": ("f16", 2, 0.5)}
PAIRS = {"f16->f32": "bf16->f32", "f16->f16": "bf16->bf16", "f16->f16 beta": "bf16->bf16 beta"}   # fp16 : bf16
BETA = {"bf16->bf16 beta": "bf16->bf16", "f16->f16 beta": "f16->f16"}                           # beta : plain


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
        ops = {"bf16": (X.bfloat16(), Y.bfloat16(), lib.b200_gemm_bf16_ex), "f16": (X.half(), Y.half(), lib.b200_gemm_f16_ex)}
        cdt = {0: torch.float32, 1: torch.bfloat16, 2: torch.float16}
        outs = {v: (torch.rand((n, n), device="cuda", generator=gen) * 2 - 1).to(cdt[ot]) for v, (_, ot, _) in VARIANTS.items()}

        def call(v, oa, ob):
            t, ot, beta = VARIANTS[v]
            A, B, fn = ops[t]
            return fn(oa, ob, n, n, n, 1.0, A.data_ptr(), n, B.data_ptr(), n, beta, outs[v].data_ptr(), n, ot, None)

        iters = max(2, int(1e13 / (2.0 * n ** 3)))
        keys = [(lay, v) for lay in LAYOUTS for v in VARIANTS]
        calls, kern, names = {k: [] for k in keys}, {k: [] for k in keys}, {}
        for lay, v in keys:                                   # warm every variant (maps, modules)
            for _ in range(2):
                assert call(v, *LAYOUTS[lay]) == 0
            names[(lay, v)] = g.last_kernel()
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for lay, v in keys:
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                lib.b200_gemm_debug_kernel_timing(1)
                s.record()
                for _ in range(iters):
                    call(v, *LAYOUTS[lay])
                e.record()
                torch.cuda.synchronize()
                ksum, cnt = g.kernel_time_ms()
                lib.b200_gemm_debug_kernel_timing(0)
                calls[(lay, v)].append(s.elapsed_time(e) / iters)
                kern[(lay, v)].append(ksum / max(cnt, 1))
        med = {k: (statistics.median(calls[k]), statistics.median(kern[k])) for k in keys}
        flop = 2.0 * n ** 3
        for lay, v in keys:
            c, k = med[(lay, v)]
            row = dict(n=n, layout=lay, variant=v, kernel_name=names[(lay, v)], call_ms=c, kernel_ms=k,
                       call_tflops=flop / c / 1e9, kernel_tflops=flop / k / 1e9,
                       spread_kernel_ms=[min(kern[(lay, v)]), max(kern[(lay, v)])])
            extra = ""
            if v in PAIRS:
                row["kernel_vs_bf16"] = med[(lay, PAIRS[v])][1] / k      # > 1: fp16 faster
                row["call_vs_bf16"] = med[(lay, PAIRS[v])][0] / c
                extra += f"  fp16:bf16 kernel {row['kernel_vs_bf16']:.3f} call {row['call_vs_bf16']:.3f}"
            if v in BETA:
                row["beta_kernel_cost"] = k / med[(lay, BETA[v])][1] - 1.0
                extra += f"  beta cost {100 * row['beta_kernel_cost']:+.1f} %"
            rows.append(row)
            print(f"N={n:5d} {lay} {v:16s} call {c:7.3f} ms {row['call_tflops']:6.1f} TFLOP/s  kernel {k:7.3f} ms "
                  f"{row['kernel_tflops']:6.1f} TFLOP/s{extra}  {names[(lay, v)]}", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
