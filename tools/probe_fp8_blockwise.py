"""Blockwise-scaled FP8 GEMM (b200_gemm_fp8_blockwise) against this library's rowwise FP8 GEMMs and its bf16 kernel.

Operands are e4m3 x e4m3 in torch's layout (row-major A, column-major B: x @ W.t(), NT), quantised from normal data as
DeepSeek-V3 does (amax / 448 per 1 x 128 group of x and per 128 x 128 block of W), bf16 out.  Shapes: m = 4096 with
(n, k) in {(7168, 2048), (2112, 7168), (24576, 1536), (7168, 16384)} (DeepSeek-V3 layer shapes), 4096^3 and 8192^3.
Arms: blockwise (1 x 128, 128 x 128) through scaled_mm; rowwise b200_gemm_fp8 promoted (fast_accum = 0) and fast
(fast_accum = 1); b200_gemm_bf16_op (NT, bf16 C) on bf16 operands of the same shape.  With --recipes, the 4096^3 shape
also times the (1 x 128, 1 x 128) and (128 x 128, 1 x 128) recipes.  Every arm is warmed up first; then the arms
alternate inside each round, each timed with CUDA events around a batch of calls (call time) and with the library's
own event pair around its GEMM kernel (kernel time); each figure is the median over rounds.

Prints the card name, power limit and max SM clock, the command line and one line per shape, and writes all of it as
JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs

OP_N, OP_T = 0, 1
OUT_BF16 = 1
SHAPES = "4096x7168x2048,4096x2112x7168,4096x24576x1536,4096x7168x16384,4096x4096x4096,8192x8192x8192"


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
    ap.add_argument("--shapes", default=SHAPES)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--recipes", action="store_true", help="also time the other two recipes at 4096^3")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    g = _libs.load_pkg()
    lib = g.lib
    info = card()
    cmd = " ".join(["python"] + sys.argv)
    print("card:", info, flush=True)
    print("command:", cmd, f"(rounds = {args.rounds})", flush=True)
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(1)
    for shape in args.shapes.split(","):
        m, n, k = (int(v) for v in shape.split("x"))
        q, mb, nb = -(-k // 128), -(-m // 128), -(-n // 128)
        x = torch.randn((m, k), device="cuda", generator=gen)
        W = torch.randn((n, k), device="cuda", generator=gen)
        sx = x.view(m, q, 128).abs().amax(dim=2) / 448                                  # (m, q)
        Wp = torch.nn.functional.pad(W, (0, 0, 0, nb * 128 - n)).view(nb, 128, q, 128)   # n may be off the grid
        sw = Wp.abs().amax(dim=(1, 3)) / 448                                           # (ceil(n / 128), q)
        xq = (x.view(m, q, 128) / sx[:, :, None]).view(m, k).to(torch.float8_e4m3fn)
        wq = (Wp / sw[:, None, :, None]).view(nb * 128, k)[:n].to(torch.float8_e4m3fn)
        del Wp
        sa_blk = sx.t().contiguous().t()                                               # outer-dim-major, as torch
        sb_blk = sw.t()                                                                # (q, ceil(n / 128))
        sa_row = sx.amax(dim=1, keepdim=True)                                          # rowwise stand-ins, same data
        sb_row = sw.amax(dim=1).repeat_interleave(128)[None, :n].contiguous()
        xb, wb = x.bfloat16(), W.bfloat16()
        del x, W
        C = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")

        def ours(sa, sb, fast=False):
            return lambda: g.scaled_mm(xq, wq.t(), sa, sb, out_dtype=torch.bfloat16, use_fast_accum=fast, out=C)

        def bf16():
            assert lib.b200_gemm_bf16_op(OP_N, OP_T, m, n, k, xb.data_ptr(), k, wb.data_ptr(), k, C.data_ptr(), n,
                                         OUT_BF16, torch.cuda.current_stream().cuda_stream) == 0

        arms = {"blk_1x128_128x128": ours(sa_blk, sb_blk), "row_promoted": ours(sa_row, sb_row),
                "row_fast": ours(sa_row, sb_row, True), "bf16": bf16}
        if args.recipes and m == n == k == 4096:
            sb_col = sb_row.expand(q, n)                                                # (q, n), stride 0 along K
            sa_128 = sx.view(mb, 128, q).amax(dim=1)                                    # (m / 128, q)
            arms["blk_1x128_1x128"] = ours(sa_blk, sb_col)
            arms["blk_128x128_1x128"] = ours(sa_128, sb_col)
        names = {}
        for a, f in arms.items():
            f(); f()
            names[a] = g.last_kernel()
        torch.cuda.synchronize()
        flop = 2.0 * m * n * k
        iters = max(5, min(100, int(4e13 / flop)))
        times = {a: [] for a in arms}
        ktimes = {a: [] for a in arms}
        for _ in range(args.rounds):
            for a, f in arms.items():
                lib.b200_gemm_debug_kernel_timing(1)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(iters):
                    f()
                e.record()
                torch.cuda.synchronize()
                times[a].append(s.elapsed_time(e) / iters)
                ms, cnt = g.kernel_time_ms()
                lib.b200_gemm_debug_kernel_timing(0)
                ktimes[a].append(ms / max(cnt, 1))
        row = dict(shape=shape, m=m, n=n, k=k, names=names, iters=iters)
        for a in arms:
            row[a] = dict(call_ms=statistics.median(times[a]), spread_ms=[min(times[a]), max(times[a])],
                          kernel_ms=statistics.median(ktimes[a]))
        rows.append(row)
        tf = lambda ms: flop / ms / 1e9
        print(f"{shape:17s} " + " | ".join(
            f"{a} {row[a]['call_ms']:.3f} ms ({tf(row[a]['call_ms']):6.1f} TF/s, kernel {row[a]['kernel_ms']:.3f} ms)"
            for a in arms) + f" | blk/promoted {row['blk_1x128_128x128']['call_ms'] / row['row_promoted']['call_ms']:.3f}"
            f" | {names['blk_1x128_128x128']}", flush=True)
        del C, xq, wq, xb, wb
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, command=cmd, rounds=args.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
