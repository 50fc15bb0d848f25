"""Strided-batched bf16 GEMM (b200_gemm_bf16_batched) against a Python loop of single-matrix calls and torch.bmm.

Shapes: attention-like batches of 128 entries, s in {512, 1024, 2048} and d in {64, 128}: QK^T (NT, m = n = s, k = d)
and PV (NN, m = s, n = d, k = s); and one large batch, 8 x 4096^3 (NN).  bf16 operands, bf16 C, alpha = 1, beta = 0.
Arms: the batched call (one launch), the loop of b200_gemm_bf16_ex calls over the entries (one launch each) and
torch.bmm (a reference point).  Per arm: whole-call time (CUDA events around a batch of calls, kernel timing off) and,
for the library's arms in separate rounds, GEMM kernel time (b200_gemm_debug_kernel_timing: per-launch event pairs,
summed over the loop's launches; those pairs also serialise the loop's launches, so only the call time compares the
arms as a caller sees them).  The arms alternate inside each round, so drift of the shared card hits them alike; each
figure is the median over rounds.  Prints the card name and power limit, the command line and the round count, one line
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

OUT_BF16 = 1


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except OSError:
        pass
    return torch.cuda.get_device_name(0) + " (power limit not readable)"


def shapes(sizes, dims, big):
    out = []
    for s in sizes:
        for d in dims:
            out.append((f"QK^T s={s} d={d}", 128, s, s, d, 1))       # (label, batch, m, n, k, op_b)
            out.append((f"PV   s={s} d={d}", 128, s, d, s, 0))
    if big:
        out.append(("8 x 4096^3", 8, 4096, 4096, 4096, 0))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="512,1024,2048")
    ap.add_argument("--dims", default="64,128")
    ap.add_argument("--no-big", action="store_true")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    g = _libs.load_pkg()
    lib = g.lib
    info = card()
    cmd = " ".join(["python"] + sys.argv)
    print("card:", info, flush=True)
    print("command:", cmd, f"(rounds = {args.rounds})", flush=True)
    rows = []
    for label, batch, m, n, k, op_b in shapes([int(x) for x in args.sizes.split(",")],
                                              [int(x) for x in args.dims.split(",")], not args.no_big):
        gen = torch.Generator(device="cuda").manual_seed(m * 7 + n * 3 + k)
        A = (torch.rand((batch, m, k), device="cuda", generator=gen) * 2 - 1).bfloat16()
        Bs = (torch.rand((batch, n, k) if op_b else (batch, k, n), device="cuda", generator=gen) * 2 - 1).bfloat16()
        Bv = Bs.transpose(1, 2) if op_b else Bs                       # the logical k x n operand of each entry
        C = torch.empty((batch, m, n), dtype=torch.bfloat16, device="cuda")
        ldb = Bs.shape[2]

        def batched():
            assert lib.b200_gemm_bf16_batched(0, op_b, m, n, k, 1.0, A.data_ptr(), k, m * k, Bs.data_ptr(), ldb,
                                              Bs.stride(0), 0.0, C.data_ptr(), n, m * n, batch, OUT_BF16, None) == 0

        def loop():
            es = A.element_size()
            for b in range(batch):
                assert lib.b200_gemm_bf16_ex(0, op_b, m, n, k, 1.0, A.data_ptr() + b * m * k * es, k,
                                             Bs.data_ptr() + b * Bs.stride(0) * es, ldb, 0.0,
                                             C.data_ptr() + b * m * n * es, n, OUT_BF16, None) == 0

        def bmm():
            torch.bmm(A, Bv, out=C)

        arms = {"batched": batched, "loop": loop, "torch.bmm": bmm}
        names = {}
        for a, f in arms.items():                                     # warm: maps, modules, cuBLAS handles
            f(); f()
            names[a] = g.last_kernel() if a != "torch.bmm" else "cuBLAS"
        torch.cuda.synchronize()
        flop = 2.0 * batch * m * n * k
        iters = min(200, max(3, int(4e12 / flop)))
        calls, kern = {a: [] for a in arms}, {a: [] for a in arms}
        for _ in range(args.rounds):
            # call time: the kernel timer off (its event pairs would sit between the loop's launches and break the
            # overlap programmatic dependent launch gives them)
            for a, f in arms.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(iters):
                    f()
                e.record()
                torch.cuda.synchronize()
                calls[a].append(s.elapsed_time(e) / iters)
            # kernel time, in rounds of its own: the library's arms with the timer on (it keeps the first 1024
            # launches: mean launch time x launches per call)
            for a in ("batched", "loop"):
                lib.b200_gemm_debug_kernel_timing(1)
                for _ in range(min(iters, max(1, 1024 // (batch if a == "loop" else 1) // 2))):
                    arms[a]()
                torch.cuda.synchronize()
                ksum, cnt = g.kernel_time_ms()
                lib.b200_gemm_debug_kernel_timing(0)
                kern[a].append(ksum / max(cnt, 1) * (batch if a == "loop" else 1))
        row = dict(shape=label, batch=batch, m=m, n=n, k=k, layout="NT" if op_b else "NN", names=names)
        for a in arms:
            row[a] = dict(call_ms=statistics.median(calls[a]), call_spread_ms=[min(calls[a]), max(calls[a])])
            if kern[a]:
                row[a].update(kernel_ms=statistics.median(kern[a]), kernel_spread_ms=[min(kern[a]), max(kern[a])])
        row["loop_over_batched_call"] = row["loop"]["call_ms"] / row["batched"]["call_ms"]
        row["loop_over_batched_kernel"] = row["loop"]["kernel_ms"] / row["batched"]["kernel_ms"]
        rows.append(row)
        tf = lambda ms: flop / ms / 1e9
        print(f"{label:22s} batched call {row['batched']['call_ms']:8.3f} ms ({tf(row['batched']['call_ms']):6.1f} TF/s) "
              f"kernel {row['batched']['kernel_ms']:8.3f} | loop call {row['loop']['call_ms']:8.3f} kernel "
              f"{row['loop']['kernel_ms']:8.3f} | bmm {row['torch.bmm']['call_ms']:8.3f} ms "
              f"({tf(row['torch.bmm']['call_ms']):6.1f} TF/s) | loop/batched call {row['loop_over_batched_call']:.2f} "
              f"kernel {row['loop_over_batched_kernel']:.2f}  {names['batched']} / {names['loop']}", flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=info, command=cmd, rounds=args.rounds, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
