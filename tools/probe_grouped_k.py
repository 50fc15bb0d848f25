"""K-grouped bf16 GEMM (b200_gemm_bf16_grouped_k) against a loop of single-matrix calls and torch._grouped_mm.

Shapes: the weight gradients of a mixture-of-experts layer with T = 16 384 routed tokens, d = 4096, d_ff = 14 336:
dW_up = dy_up^T x (m = d_ff, n = d) and dW_down = dy_down^T h (m = d, n = d_ff), with G = 8 and G = 64 experts, each
with a balanced routing (equal groups) and a skewed one (group sizes proportional to 1 / rank, Zipf s = 1).  dy is a
row-major (T, m) gradient passed as dy.t(), so A is read as op_a = T; x is a row-major (T, n) activation, op_b = N.
bf16 operands, bf16 C, alpha = 1, beta = 0.  Arms: the K-grouped call (one launch, offsets on the device), the loop of
b200_gemm_bf16_ex calls over the groups with the offsets already on the host (one launch per group; an empty group is
the k = 0 call, which writes its zeros), and torch._grouped_mm(dy.t(), x, offs=offs).  Every shape is warmed up first;
then the arms alternate inside each round, each timed with CUDA events around a batch of calls, and each figure is the
median over rounds.  For each shape it also prints the least time the data sheet allows (989 TFLOP/s dense bf16,
3.35 TB/s HBM3, H100 SXM at 700 W) from the FLOPs 2 T m n and the bytes T (m + n) * 2 read plus G m n * 2 written,
and which of the two bounds it.  Prints the card name, power limit and max SM clock, the command line and one line
per shape, and writes all of it as JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs

OUT_BF16, OP_N, OP_T = 1, 0, 1
PEAK_FLOPS, PEAK_BYTES = 989e12, 3.35e12     # H100 SXM data sheet: dense bf16, HBM3


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except OSError:
        pass
    return torch.cuda.get_device_name(0) + " (power limit not readable)"


def routing(total, groups, skew):
    """Group sizes summing to total: equal, or proportional to 1 / (rank + 1)."""
    w = [1.0 / (i + 1) if skew else 1.0 for i in range(groups)]
    sizes = [int(total * x / sum(w)) for x in w]
    sizes[0] += total - sum(sizes)
    return sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=16384)
    ap.add_argument("--d", type=int, default=4096)
    ap.add_argument("--dff", type=int, default=14336)
    ap.add_argument("--groups", default="8,64")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    g = _libs.load_pkg()
    lib = g.lib
    info = card()
    cmd = " ".join(["python"] + sys.argv)
    print("card:", info, flush=True)
    print("command:", cmd, f"(rounds = {args.rounds})", flush=True)
    T = args.tokens
    cases = []
    for G in [int(x) for x in args.groups.split(",")]:
        for skew in (False, True):
            for proj, m, n in (("up", args.dff, args.d), ("down", args.d, args.dff)):
                cases.append((f"dW_{proj:4s} G={G:2d} {'zipf' if skew else 'even'}", G, skew, m, n))
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(1)
    for label, G, skew, m, n in cases:
        sizes = routing(T, G, skew)
        ends = [sum(sizes[:i + 1]) for i in range(G)]
        offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
        dy = ((torch.rand((T, m), device="cuda", generator=gen) * 2 - 1) / 16).bfloat16()
        x = (torch.rand((T, n), device="cuda", generator=gen) * 2 - 1).bfloat16()
        C = torch.empty((G, m, n), dtype=torch.bfloat16, device="cuda")
        es = x.element_size()

        def grouped_k():
            assert lib.b200_gemm_bf16_grouped_k(OP_T, OP_N, m, n, T, 1.0, dy.data_ptr(), m, x.data_ptr(), n,
                                                offs.data_ptr(), G, 0.0, C.data_ptr(), n, m * n, OUT_BF16, None) == 0

        def loop():
            lo = 0
            for i, hi in enumerate(ends):
                assert lib.b200_gemm_bf16_ex(OP_T, OP_N, m, n, hi - lo, 1.0, dy.data_ptr() + lo * m * es, m,
                                             x.data_ptr() + lo * n * es, n, 0.0, C.data_ptr() + i * m * n * es, n,
                                             OUT_BF16, None) == 0
                lo = hi

        def torch_grouped():
            torch._grouped_mm(dy.t(), x, offs=offs)

        arms = {"grouped_k": grouped_k, "loop": loop, "torch": torch_grouped}
        names = {}
        for a, f in arms.items():
            f(); f()
            names[a] = g.last_kernel() if a != "torch" else "torch._grouped_mm"
        torch.cuda.synchronize()
        flop = 2.0 * T * m * n
        nbytes = 2.0 * (T * (m + n) + G * m * n)
        t_flop, t_bytes = flop / PEAK_FLOPS * 1e3, nbytes / PEAK_BYTES * 1e3
        bound = "MMA" if t_flop >= t_bytes else "HBM write"
        iters = max(3, min(50, int(2e13 / flop)))
        times = {a: [] for a in arms}
        for _ in range(args.rounds):
            for a, f in arms.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(iters):
                    f()
                e.record()
                torch.cuda.synchronize()
                times[a].append(s.elapsed_time(e) / iters)
        row = dict(shape=label, groups=G, sizes=sizes, m=m, n=n, tokens=T, names=names,
                   bound=dict(kind=bound, flop_ms=t_flop, bytes_ms=t_bytes))
        for a in arms:
            row[a] = dict(call_ms=statistics.median(times[a]), spread_ms=[min(times[a]), max(times[a])])
        row["loop_over_grouped_k"] = row["loop"]["call_ms"] / row["grouped_k"]["call_ms"]
        row["torch_over_grouped_k"] = row["torch"]["call_ms"] / row["grouped_k"]["call_ms"]
        rows.append(row)
        del C
        tf = lambda ms: flop / ms / 1e9
        print(f"{label:22s} grouped_k {row['grouped_k']['call_ms']:7.3f} ms ({tf(row['grouped_k']['call_ms']):5.1f} TF/s) | "
              f"loop {row['loop']['call_ms']:7.3f} ms ({tf(row['loop']['call_ms']):5.1f}) | torch "
              f"{row['torch']['call_ms']:7.3f} ms ({tf(row['torch']['call_ms']):5.1f}) | loop/grouped_k "
              f"{row['loop_over_grouped_k']:.2f} torch/grouped_k {row['torch_over_grouped_k']:.2f} | bound {bound} "
              f"(flop {t_flop:.3f} ms, bytes {t_bytes:.3f} ms)  {names['grouped_k']}", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, command=cmd, rounds=args.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
