"""Grouped bf16 GEMM (b200_gemm_bf16_grouped) against a loop of single-matrix calls and torch._grouped_mm.

Shapes: the projections of a mixture-of-experts layer, 16 384 routed rows, d = 4096, d_ff = 14 336: the up-projection
(n = d_ff, k = d) and the down-projection (n = d, k = d_ff), with G = 8 and G = 64 experts, each with a balanced routing
(equal groups) and a skewed one (group sizes proportional to 1 / rank, Zipf s = 1).  The weights are (G, n, k)
parameters passed as W.transpose(-2, -1), so B is read as op_b = T.  bf16 operands, bf16 C, alpha = 1, beta = 0.
Arms: the grouped call (one launch, offsets on the device), the loop of b200_gemm_bf16_ex calls over the groups with the
offsets already on the host (one launch per non-empty group), and torch._grouped_mm.  Every shape is warmed up first;
then the arms alternate inside each round, each timed with CUDA events around a batch of calls, and each figure is the
median over rounds.  Prints the card name, power limit and max SM clock, the command line and one line per shape, and
writes all of it as JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs

OUT_BF16, OP_T = 1, 1


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
    ap.add_argument("--rows", type=int, default=16384)
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
    cases = []
    for G in [int(x) for x in args.groups.split(",")]:
        for skew in (False, True):
            for proj, n, k in (("up", args.dff, args.d), ("down", args.d, args.dff)):
                cases.append((f"{proj:4s} G={G:2d} {'zipf' if skew else 'even'}", G, skew, n, k))
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(1)
    weights = {}
    for label, G, skew, n, k in cases:
        total = args.rows
        sizes = routing(total, G, skew)
        ends = [sum(sizes[:i + 1]) for i in range(G)]
        offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
        x = (torch.rand((total, k), device="cuda", generator=gen) * 2 - 1).bfloat16()
        if (G, n, k) not in weights:
            weights.clear()
            weights[(G, n, k)] = ((torch.rand((G, n, k), device="cuda", generator=gen) * 2 - 1) / 16).bfloat16()
        W = weights[(G, n, k)]
        Bt = W.transpose(-2, -1)
        C = torch.empty((total, n), dtype=torch.bfloat16, device="cuda")
        es = x.element_size()

        def grouped():
            assert lib.b200_gemm_bf16_grouped(OP_T, total, n, k, 1.0, x.data_ptr(), k, W.data_ptr(), k, n * k,
                                              offs.data_ptr(), G, 0.0, C.data_ptr(), n, OUT_BF16, None) == 0

        def loop():
            lo = 0
            for i, hi in enumerate(ends):
                if hi > lo:
                    assert lib.b200_gemm_bf16_ex(0, OP_T, hi - lo, n, k, 1.0, x.data_ptr() + lo * k * es, k,
                                                 W.data_ptr() + i * n * k * es, k, 0.0, C.data_ptr() + lo * n * es, n,
                                                 OUT_BF16, None) == 0
                lo = hi

        def torch_grouped():
            torch._grouped_mm(x, Bt, offs=offs)

        arms = {"grouped": grouped, "loop": loop, "torch": torch_grouped}
        names = {}
        for a, f in arms.items():
            f(); f()
            names[a] = g.last_kernel() if a != "torch" else "torch._grouped_mm"
        torch.cuda.synchronize()
        flop = 2.0 * total * n * k
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
        row = dict(shape=label, groups=G, sizes=sizes, n=n, k=k, total_m=total, names=names)
        for a in arms:
            row[a] = dict(call_ms=statistics.median(times[a]), spread_ms=[min(times[a]), max(times[a])])
        row["loop_over_grouped"] = row["loop"]["call_ms"] / row["grouped"]["call_ms"]
        row["torch_over_grouped"] = row["torch"]["call_ms"] / row["grouped"]["call_ms"]
        rows.append(row)
        tf = lambda ms: flop / ms / 1e9
        print(f"{label:18s} grouped {row['grouped']['call_ms']:7.3f} ms ({tf(row['grouped']['call_ms']):5.1f} TF/s) | "
              f"loop {row['loop']['call_ms']:7.3f} ms ({tf(row['loop']['call_ms']):5.1f}) | torch "
              f"{row['torch']['call_ms']:7.3f} ms ({tf(row['torch']['call_ms']):5.1f}) | loop/grouped "
              f"{row['loop_over_grouped']:.2f} torch/grouped {row['torch_over_grouped']:.2f}  {names['grouped']}",
              flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, command=cmd, rounds=args.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
