"""FP8 GEMM (b200_gemm_fp8) against torch._scaled_mm and this library's bf16 kernel, and the tensor core's retained FP8
accumulation precision.

Timing: e4m3 x e4m3 operands, rowwise scales, bf16 out, torch's layout (row-major A, column-major B: x @ W.t(), NT).
Shapes 4096^3, 8192^3 and the MLP shape m = 8192, n = 16384, k = 4096.  Arms: b200_gemm_fp8 promoted (fast_accum = 0)
and fast (fast_accum = 1), torch._scaled_mm with use_fast_accum False and True on the same tensors, and
b200_gemm_bf16_op (NT, bf16 C) on bf16 operands of the same shape.  Every shape is warmed up first; then the arms
alternate inside each round, each timed with CUDA events around a batch of calls (call time), and for this library's
arms also with the library's own event pair around its GEMM kernel (kernel time); each figure is the median over rounds.

Precision: the fp32 result of a crafted sum 2^e + 1 (an e4m3 power of two times an e5m2 one, then 1 * 1, in the same
MMA or in a later one) tells whether the tensor core's accumulation keeps e + 1 bits; the largest such e + 1 is the
retained precision.  Ordinary finite inputs only.

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
FP8_E4M3, FP8_E5M2 = 0, 1
OUT_F32, OUT_BF16 = 0, 1
PEAK_FP8, PEAK_BF16 = 1979e12, 989e12     # H100 SXM data sheet, dense, 700 W


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except OSError:
        pass
    return torch.cuda.get_device_name(0) + " (power limit not readable)"


def retained_bits(lib, split):
    """Largest p with 2^(p-1) + 1 exact in the fp32 result (the +1 at K index `split`; fast_accum = 1, k = 128)."""
    k = 128
    one = torch.ones(1, device="cuda")
    C = torch.empty((1, 1), device="cuda")
    for p in range(1, 25):
        a = torch.zeros((1, k), device="cuda")
        b = torch.zeros((1, k), device="cuda")
        e1 = min(p, 8)
        a[0, 0], b[0, 0] = 2.0 ** e1, 2.0 ** (p - e1)
        a[0, split], b[0, split] = 1.0, 1.0
        A, B = a.to(torch.float8_e4m3fn), b.to(torch.float8_e5m2)
        assert lib.b200_gemm_fp8(OP_N, OP_T, FP8_E4M3, FP8_E5M2, 1, 1, k, A.data_ptr(), k, B.data_ptr(), k,
                                 one.data_ptr(), 0, one.data_ptr(), 0, None, C.data_ptr(), 1, OUT_F32, 1, None) == 0
        if C.item() - 2.0 ** p != 1.0:
            return p
    return 25


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="4096x4096x4096,8192x8192x8192,8192x16384x4096")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    g = _libs.load_pkg()
    lib = g.lib
    info = card()
    cmd = " ".join(["python"] + sys.argv)
    print("card:", info, flush=True)
    print("command:", cmd, f"(rounds = {args.rounds})", flush=True)
    bits = dict(inside_one_mma=retained_bits(lib, 1), across_mmas=retained_bits(lib, 64))
    print("retained FP8 accumulation bits:", bits, flush=True)
    rows = []
    gen = torch.Generator(device="cuda").manual_seed(1)
    for shape in args.shapes.split(","):
        m, n, k = (int(v) for v in shape.split("x"))
        x = torch.randn((m, k), device="cuda", generator=gen)
        W = torch.randn((n, k), device="cuda", generator=gen)
        sx = x.abs().amax(dim=1, keepdim=True) / 448
        sw = W.abs().amax(dim=1, keepdim=True) / 448
        xq, wq = (x / sx).to(torch.float8_e4m3fn), (W / sw).to(torch.float8_e4m3fn)
        swt = sw.t().contiguous()
        xb, wb = x.bfloat16(), W.bfloat16()
        del x, W
        C = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")

        def ours(fast):
            return lambda: g.scaled_mm(xq, wq.t(), sx, swt, out_dtype=torch.bfloat16, use_fast_accum=fast, out=C)

        def torch_arm(fast):
            return lambda: torch._scaled_mm(xq, wq.t(), sx, swt, out_dtype=torch.bfloat16, use_fast_accum=fast)

        def bf16():
            assert lib.b200_gemm_bf16_op(OP_N, OP_T, m, n, k, xb.data_ptr(), k, wb.data_ptr(), k, C.data_ptr(), n,
                                         OUT_BF16, torch.cuda.current_stream().cuda_stream) == 0

        arms = {"fp8_promoted": ours(False), "fp8_fast": ours(True), "torch_fp8": torch_arm(False),
                "torch_fp8_fast": torch_arm(True), "bf16": bf16}
        ours_arms = ("fp8_promoted", "fp8_fast", "bf16")
        names = {}
        for a, f in arms.items():
            f(); f()
            names[a] = g.last_kernel() if a in ours_arms else "torch._scaled_mm"
        torch.cuda.synchronize()
        flop = 2.0 * m * n * k
        iters = max(5, min(100, int(4e13 / flop)))
        times = {a: [] for a in arms}
        ktimes = {a: [] for a in ours_arms}
        for _ in range(args.rounds):
            for a, f in arms.items():
                if a in ours_arms:
                    lib.b200_gemm_debug_kernel_timing(1)
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(iters):
                    f()
                e.record()
                torch.cuda.synchronize()
                times[a].append(s.elapsed_time(e) / iters)
                if a in ours_arms:
                    ms, cnt = g.kernel_time_ms()
                    lib.b200_gemm_debug_kernel_timing(0)
                    ktimes[a].append(ms / max(cnt, 1))
        row = dict(shape=shape, m=m, n=n, k=k, names=names, iters=iters)
        for a in arms:
            row[a] = dict(call_ms=statistics.median(times[a]), spread_ms=[min(times[a]), max(times[a])])
            if a in ours_arms:
                row[a]["kernel_ms"] = statistics.median(ktimes[a])
        rows.append(row)
        tf = lambda ms: flop / ms / 1e9
        print(f"{shape:17s} " + " | ".join(
            f"{a} {row[a]['call_ms']:.3f} ms ({tf(row[a]['call_ms']):6.1f} TF/s"
            + (f", kernel {row[a]['kernel_ms']:.3f} ms {tf(row[a]['kernel_ms']):6.1f}" if a in ours_arms else "") + ")"
            for a in arms) + f" | promoted/fast {row['fp8_promoted']['call_ms'] / row['fp8_fast']['call_ms']:.3f}"
            f" | bf16/fast {row['bf16']['call_ms'] / row['fp8_fast']['call_ms']:.3f}"
            f" | {names['fp8_promoted']} {names['fp8_fast']}", flush=True)
        del C, xq, wq, xb, wb
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, command=cmd, rounds=args.rounds, retained_bits=bits, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
