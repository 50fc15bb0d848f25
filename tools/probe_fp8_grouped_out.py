"""The fused FP8 output of the grouped blockwise FP8 GEMM (b200_gemm_fp8_blockwise_grouped_q8) against the unfused
chain it replaces, the bf16-output call alone, and a loop of single-matrix b200_gemm_fp8_blockwise_q8 calls.

Shapes: DeepSeek-V3's routed experts with 16 384 routed rows, d = 7168, expert d_ff = 2048: n = 4096, k = 7168 (the
up projection, gate and up together) and n = 7168, k = 2048 (the down projection), with G = 8, 32 and 256 experts,
each with a balanced routing and a skewed one (group sizes proportional to 1 / rank).  Operands are quantised as
DeepSeek-V3 does (x per 1 x 128, each expert's weight per 128 x 128; probe_fp8_blockwise_grouped.quantised_weights).
Arms:
  q8        b200_gemm_fp8_blockwise_grouped_q8, no activation: C e4m3 and its 1 x 128 scales in one launch
  q8_gelu   the same with GELU
  unfused   b200_gemm_fp8_blockwise_grouped with bf16 C, then the same 1 x 128 quantisation in torch ops
  bf16      b200_gemm_fp8_blockwise_grouped with bf16 C alone
  loop_q8   b200_gemm_fp8_blockwise_q8 per non-empty group, the offsets already on the host
and, at the first shape only, row_q8: b200_gemm_fp8_grouped_q8 promoted (rowwise scales) on the same FP8 bytes.
Every shape is warmed up first; the arms then alternate inside each round, each timed with CUDA events around a batch
of calls, and each figure is the median over rounds with the min / max beside it.  The HBM bytes each arm must move
are counted from the shapes (operands read once, C and scales written, the unfused chain's bf16 C written and read
back).  Prints the card name, power limit and max SM clock, the command line and one line per shape, and writes all of
it as JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _libs
from probe_fp8_blockwise_grouped import quantised_weights
from probe_grouped import card, routing

E4M3, OUT_BF16, OP_N, OP_T, ACT_NONE, ACT_GELU = 0, 1, 0, 1, 0, 2


def hbm_bytes(total, n, k, G, groups_used):
    """Bytes each arm must move: A and the used experts' B read once, C (and its scales) written; scales of A / B are
    small and counted too."""
    q, qn = k // 128, -(-n // 128)
    inputs = total * k + groups_used * n * k + 4 * (total * q + groups_used * q * qn)
    fp8_out = total * n + 4 * total * qn
    return dict(q8=inputs + fp8_out, bf16=inputs + 2 * total * n,
                unfused=inputs + 2 * total * n + 2 * total * n + fp8_out)


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
        for n, k in ((2 * args.dff, args.d), (args.d, args.dff)):
            for skew in (False, True):
                cases.append((f"n={n:5d} k={k:5d} G={G:3d} {'zipf' if skew else 'even'}", G, skew, n, k))
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(1)
    weights = {}
    for ci, (label, G, skew, n, k) in enumerate(cases):
        total = args.rows
        q, qn = k // 128, -(-n // 128)
        sizes = routing(total, G, skew)
        ends = [sum(sizes[:i + 1]) for i in range(G)]
        offs = torch.tensor(ends, dtype=torch.int32, device="cuda")
        x = torch.randn((total, k), device="cuda", generator=gen)
        sx = (x.view(total, q, 128).abs().amax(dim=2) / 448).clamp_min(1e-12)
        xq = (x.view(total, q, 128) / sx[:, :, None]).view(total, k).to(torch.float8_e4m3fn)
        del x
        sa = sx.t().contiguous().t()                       # (total, q), outer-dim-major
        if (G, n, k) not in weights:
            weights.clear()
            torch.cuda.empty_cache()
            Wq, sw, _ = quantised_weights(G, n, k, gen)
            weights[(G, n, k)] = (Wq, sw)
        Wq, sb = weights[(G, n, k)]                        # sb (G, q, qn)
        sa_r, sb_r = torch.ones(total, device="cuda"), torch.ones((G, n), device="cuda")
        C16 = torch.empty((total, n), dtype=torch.bfloat16, device="cuda")
        C8 = torch.empty((total, n), dtype=torch.uint8, device="cuda")
        SC = torch.empty((total, qn), device="cuda")

        def q8(act=ACT_NONE):
            assert lib.b200_gemm_fp8_blockwise_grouped_q8(
                E4M3, E4M3, total, n, k, xq.data_ptr(), k, Wq.data_ptr(), k, n * k, offs.data_ptr(), G, sa.data_ptr(),
                sa.stride(0), sa.stride(1), sb.data_ptr(), 128, sb.stride(1), sb.stride(2), sb.stride(0), act, E4M3,
                C8.data_ptr(), n, SC.data_ptr(), qn, 1, None) == 0

        def bf16():
            assert lib.b200_gemm_fp8_blockwise_grouped(E4M3, E4M3, total, n, k, xq.data_ptr(), k, Wq.data_ptr(), k,
                                                       n * k, offs.data_ptr(), G, sa.data_ptr(), sa.stride(0),
                                                       sa.stride(1), sb.data_ptr(), 128, sb.stride(1), sb.stride(2),
                                                       sb.stride(0), C16.data_ptr(), n, OUT_BF16, None) == 0

        def unfused():
            bf16()
            blk = C16.view(total, qn, 128).float()
            d = blk.abs().amax(dim=2) / 448
            d = torch.where(d == 0, torch.ones_like(d), d)
            SC.copy_(d)
            C8.view(torch.float8_e4m3fn).copy_((blk / d[:, :, None]).clamp(-448, 448).view(total, n))

        def loop_q8():
            lo = 0
            for i, hi in enumerate(ends):
                if hi > lo:
                    assert lib.b200_gemm_fp8_blockwise_q8(
                        OP_N, OP_T, E4M3, E4M3, hi - lo, n, k, xq.data_ptr() + lo * k, k, Wq.data_ptr() + i * n * k, k,
                        sa.data_ptr() + 4 * lo, 1, sa.stride(0), sa.stride(1), sb.data_ptr() + 4 * i * sb.stride(0),
                        128, sb.stride(1), sb.stride(2), None, ACT_NONE, E4M3, C8.data_ptr() + lo * n, n, None,
                        SC.data_ptr() + 4 * lo * qn, qn, 1, None) == 0
                lo = hi

        def row_q8():
            assert lib.b200_gemm_fp8_grouped_q8(E4M3, E4M3, total, n, k, xq.data_ptr(), k, Wq.data_ptr(), k, n * k,
                                                offs.data_ptr(), G, sa_r.data_ptr(), sb_r.data_ptr(), n, ACT_NONE, 0,
                                                E4M3, C8.data_ptr(), n, SC.data_ptr(), qn, 1, None) == 0

        arms = {"q8": q8, "q8_gelu": lambda: q8(ACT_GELU), "unfused": unfused, "bf16": bf16, "loop_q8": loop_q8}
        if ci == 0:
            arms["row_q8"] = row_q8
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
        used = sum(1 for s_ in sizes if s_ > 0)
        nbytes = hbm_bytes(total, n, k, G, used)
        row = dict(shape=label, groups=G, sizes=sizes, n=n, k=k, total_m=total, names=names, hbm_bytes=nbytes)
        for a in arms:
            row[a] = dict(call_ms=statistics.median(times[a]), spread_ms=[min(times[a]), max(times[a])])
        rows.append(row)
        parts = [f"{a} {row[a]['call_ms']:7.3f} [{row[a]['spread_ms'][0]:.3f}-{row[a]['spread_ms'][1]:.3f}]"
                 for a in arms]
        print(f"{label} ms: " + " | ".join(parts) +
              f" | q8/bf16 {row['q8']['call_ms'] / row['bf16']['call_ms']:.3f}"
              f" q8/unfused {row['q8']['call_ms'] / row['unfused']['call_ms']:.3f}"
              f" | HBM MB q8 {nbytes['q8'] / 1e6:.0f} bf16 {nbytes['bf16'] / 1e6:.0f} unfused {nbytes['unfused'] / 1e6:.0f}",
              flush=True)
        del xq, sx, sa, C16, C8, SC
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, command=cmd, rounds=args.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
