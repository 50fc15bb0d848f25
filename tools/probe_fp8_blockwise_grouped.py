"""Grouped blockwise FP8 GEMM (b200_gemm_fp8_blockwise_grouped) against a loop of single-matrix blockwise calls, the
grouped rowwise FP8 GEMM and the grouped bf16 GEMM.

Shapes: DeepSeek-V3's routed experts, d = 7168, expert d_ff = 2048, with 16 384 routed rows: the up projection
(n = 2 * d_ff = 4096, gate and up together, k = d) and the down projection (n = d, k = d_ff), with G = 8, 32 and 256
experts, each with a balanced routing and a skewed one (group sizes proportional to 1 / rank, Zipf s = 1).  Operands are
quantised to e4m3 as DeepSeek-V3 does: x per 1 x 128 group (amax / 448; scale_a (rows, k / 128) outer-dim-major, as
torch takes it) and each expert's weight per 128 x 128 block (scale_b (G, k / 128, n / 128)); bf16 C.
Arms: the grouped blockwise call (one launch, offsets on the device); the loop of b200_gemm_fp8_blockwise (N, T) calls
over the groups with the offsets already on the host (one launch per non-empty group); b200_gemm_fp8_grouped promoted
(rowwise scales) on the same FP8 bytes; and b200_gemm_bf16_grouped on bf16 copies of the unquantised operands.  Every
shape is warmed up first; then the arms alternate inside each round, each timed with CUDA events around a batch of
calls, and each figure is the median over rounds with the min / max beside it.  Prints the card name, power limit and
max SM clock, the command line and one line per shape, and writes all of it as JSON to the file named by --out."""
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


def quantised_weights(G, n, k, gen, chunk=8):
    """e4m3 (G, n, k) weights quantised per 128 x 128 block, their scales (G, k / 128, n / 128) and bf16 copies,
    generated a few experts at a time."""
    Wq = torch.empty((G, n, k), dtype=torch.float8_e4m3fn, device="cuda")
    Wb = torch.empty((G, n, k), dtype=torch.bfloat16, device="cuda")
    sw = torch.empty((G, n // 128, k // 128), device="cuda")
    for g0 in range(0, G, chunk):
        g1 = min(G, g0 + chunk)
        W = torch.randn((g1 - g0, n, k), device="cuda", generator=gen) / 16
        blk = W.view(g1 - g0, n // 128, 128, k // 128, 128)
        s = (blk.abs().amax(dim=(2, 4)) / 448).clamp_min(1e-12)
        Wq[g0:g1] = (blk / s[:, :, None, :, None]).view(W.shape).to(torch.float8_e4m3fn)
        Wb[g0:g1] = W.bfloat16()
        sw[g0:g1] = s
        del W, blk
    return Wq, sw.transpose(1, 2), Wb


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rows", type=int, default=16384)
    ap.add_argument("--d", type=int, default=7168)
    ap.add_argument("--dff", type=int, default=2048)
    ap.add_argument("--groups", default="8,32,256")
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
        for proj, n, k in (("up", 2 * args.dff, args.d), ("down", args.d, args.dff)):
            for skew in (False, True):
                cases.append((f"{proj:4s} G={G:3d} {'zipf' if skew else 'even'}", G, skew, n, k))
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(1)
    weights = {}
    for label, G, skew, n, k in cases:
        total = args.rows
        q, nb = k // 128, n // 128
        sizes = routing(total, G, skew)
        ends = [sum(sizes[:i + 1]) for i in range(G)]
        offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
        x = torch.randn((total, k), device="cuda", generator=gen)
        sx = (x.view(total, q, 128).abs().amax(dim=2) / 448).clamp_min(1e-12)
        xq = (x.view(total, q, 128) / sx[:, :, None]).view(total, k).to(torch.float8_e4m3fn)
        xb = x.bfloat16()
        del x
        sa = sx.t().contiguous().t()                       # (total, q), outer-dim-major: strides (1, total)
        if (G, n, k) not in weights:
            weights.clear()
            torch.cuda.empty_cache()
            weights[(G, n, k)] = quantised_weights(G, n, k, gen)
        Wq, sb, Wb = weights[(G, n, k)]                    # sb (G, q, nb), strides (nb * q, 1, q)
        sa_r, sb_r = torch.ones(total, device="cuda"), torch.ones((G, n), device="cuda")
        C = torch.empty((total, n), dtype=torch.bfloat16, device="cuda")

        def grouped_blk():
            assert lib.b200_gemm_fp8_blockwise_grouped(E4M3, E4M3, total, n, k, xq.data_ptr(), k, Wq.data_ptr(), k,
                                                       n * k, offs.data_ptr(), G, sa.data_ptr(), sa.stride(0),
                                                       sa.stride(1), sb.data_ptr(), 128, sb.stride(1), sb.stride(2),
                                                       sb.stride(0), C.data_ptr(), n, OUT_BF16, None) == 0

        def loop_blk():
            lo = 0
            for i, hi in enumerate(ends):
                if hi > lo:
                    assert lib.b200_gemm_fp8_blockwise(OP_N, OP_T, E4M3, E4M3, hi - lo, n, k, xq.data_ptr() + lo * k, k,
                                                       Wq.data_ptr() + i * n * k, k, sa.data_ptr() + 4 * lo, 1,
                                                       sa.stride(0), sa.stride(1), sb.data_ptr() + 4 * i * sb.stride(0),
                                                       128, sb.stride(1), sb.stride(2), None, C.data_ptr() + 2 * lo * n,
                                                       n, OUT_BF16, None) == 0
                lo = hi

        def grouped_rowwise():
            assert lib.b200_gemm_fp8_grouped(E4M3, E4M3, total, n, k, xq.data_ptr(), k, Wq.data_ptr(), k, n * k,
                                             offs.data_ptr(), G, sa_r.data_ptr(), sb_r.data_ptr(), n, C.data_ptr(), n,
                                             OUT_BF16, 0, None) == 0

        def bf16_grouped():
            assert lib.b200_gemm_bf16_grouped(OP_T, total, n, k, 1.0, xb.data_ptr(), k, Wb.data_ptr(), k, n * k,
                                              offs.data_ptr(), G, 0.0, C.data_ptr(), n, OUT_BF16, None) == 0

        arms = {"grp_blk": grouped_blk, "loop_blk": loop_blk, "grp_rowwise_acc": grouped_rowwise, "bf16_grp": bf16_grouped}
        names = {}
        for a, f in arms.items():
            f(); f()
            names[a] = g.last_kernel()
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
        rows.append(row)
        tf = lambda ms: flop / ms / 1e9
        parts = [f"{a} {row[a]['call_ms']:7.3f} ms [{row[a]['spread_ms'][0]:.3f}-{row[a]['spread_ms'][1]:.3f}] "
                 f"({tf(row[a]['call_ms']):6.1f} TF/s)" for a in arms]
        ratio = row["loop_blk"]["call_ms"] / row["grp_blk"]["call_ms"]
        print(f"{label:18s} " + " | ".join(parts) + f" | loop_blk/grp_blk {ratio:.3f}", flush=True)
        del xq, xb, sx, sa, C
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, command=cmd, rounds=args.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
