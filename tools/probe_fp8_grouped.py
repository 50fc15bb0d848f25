"""Grouped FP8 GEMM (b200_gemm_fp8_grouped) against a loop of single-matrix FP8 calls, torch._scaled_grouped_mm and the
grouped bf16 GEMM.

Shapes: those of tools/probe_grouped.py, the projections of a mixture-of-experts layer with 16 384 routed rows,
d = 4096, d_ff = 14 336: the up-projection (n = d_ff, k = d) and the down-projection (n = d, k = d_ff), with G = 8 and
G = 64 experts, each with a balanced routing and a skewed one (group sizes proportional to 1 / rank, Zipf s = 1).  e4m3
operands with rowwise scales (scale_a one per routed row, scale_b one per column of each expert), bf16 C; the weights
are (G, n, k) parameters passed as W.transpose(-2, -1).
Arms: the grouped call, promoted and fast (one launch, offsets on the device); the loop of b200_gemm_fp8 (N, T) calls
over the groups with the offsets already on the host (one launch per non-empty group), promoted and fast;
torch._scaled_grouped_mm with use_fast_accum False and True (reported as refused where torch has no kernel); and
b200_gemm_bf16_grouped on bf16 copies of the same operands.  Every shape is warmed up first; then the arms alternate
inside each round, each timed with CUDA events around a batch of calls, and each figure is the median over rounds with
the min / max beside it.  Prints the card name, power limit and max SM clock, the command line and one line per shape,
and writes all of it as JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _libs
from probe_grouped import card, routing

E4M3, OUT_BF16, OP_N, OP_T = 0, 1, 0, 1


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
        x = torch.randn((total, k), device="cuda", generator=gen)
        sa = (x.abs().amax(dim=1) / 448.0).clamp(min=1e-12)
        xq = (x / sa[:, None]).to(torch.float8_e4m3fn)
        xb = x.bfloat16()
        del x
        if (G, n, k) not in weights:
            weights.clear()
            W = torch.randn((G, n, k), device="cuda", generator=gen) / 16
            sb = (W.abs().amax(dim=2) / 448.0).clamp(min=1e-12)
            weights[(G, n, k)] = ((W / sb[:, :, None]).to(torch.float8_e4m3fn), sb.contiguous(), W.bfloat16())
            del W
        Wq, sb, Wb = weights[(G, n, k)]
        Bt = Wq.transpose(-2, -1)
        C = torch.empty((total, n), dtype=torch.bfloat16, device="cuda")

        def grouped(fast):
            assert lib.b200_gemm_fp8_grouped(E4M3, E4M3, total, n, k, xq.data_ptr(), k, Wq.data_ptr(), k, n * k,
                                             offs.data_ptr(), G, sa.data_ptr(), sb.data_ptr(), n, C.data_ptr(), n,
                                             OUT_BF16, fast, None) == 0

        def loop(fast):
            lo = 0
            for i, hi in enumerate(ends):
                if hi > lo:
                    assert lib.b200_gemm_fp8(OP_N, OP_T, E4M3, E4M3, hi - lo, n, k, xq.data_ptr() + lo * k, k,
                                             Wq.data_ptr() + i * n * k, k, sa.data_ptr() + 4 * lo, 1,
                                             sb.data_ptr() + 4 * i * n, 1, None, C.data_ptr() + 2 * lo * n, n,
                                             OUT_BF16, fast, None) == 0
                lo = hi

        def torch_scaled(fast):
            torch._scaled_grouped_mm(xq, Bt, sa, sb, offs=offs, out_dtype=torch.bfloat16, use_fast_accum=bool(fast))

        def bf16_grouped():
            assert lib.b200_gemm_bf16_grouped(OP_T, total, n, k, 1.0, xb.data_ptr(), k, Wb.data_ptr(), k, n * k,
                                              offs.data_ptr(), G, 0.0, C.data_ptr(), n, OUT_BF16, None) == 0

        arms = {"grp_acc": lambda: grouped(0), "grp_fast": lambda: grouped(1), "loop_acc": lambda: loop(0),
                "loop_fast": lambda: loop(1), "torch_acc": lambda: torch_scaled(0), "torch_fast": lambda: torch_scaled(1),
                "bf16_grp": bf16_grouped}
        names, refused = {}, {}
        for a, f in list(arms.items()):
            try:
                f(); f()
            except RuntimeError as e:                    # torch without a kernel for this call on this stack
                refused[a] = str(e).splitlines()[0][:200]
                del arms[a]
                continue
            names[a] = g.last_kernel() if not a.startswith("torch") else "torch._scaled_grouped_mm"
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
        row = dict(shape=label, groups=G, sizes=sizes, n=n, k=k, total_m=total, names=names, refused=refused)
        for a in arms:
            row[a] = dict(call_ms=statistics.median(times[a]), spread_ms=[min(times[a]), max(times[a])])
        rows.append(row)
        tf = lambda ms: flop / ms / 1e9
        parts = [f"{a} {row[a]['call_ms']:7.3f} ms ({tf(row[a]['call_ms']):6.1f} TF/s)" for a in arms]
        ratios = f"loop_fast/grp_fast {row['loop_fast']['call_ms'] / row['grp_fast']['call_ms']:.3f}"
        if "torch_fast" in row:
            ratios += f" torch_fast/grp_fast {row['torch_fast']['call_ms'] / row['grp_fast']['call_ms']:.3f}"
        print(f"{label:18s} " + " | ".join(parts) + " | " + ratios + (f" | refused {sorted(refused)}" if refused else ""),
              flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, command=cmd, rounds=args.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
