"""Blockwise FP8 quantisers (b200_fp8_quantize) against the torch-ops quantisation they replace and a device copy.

Shapes (bf16 inputs, e4m3 outputs, every arm writing the transposed copy too):
  act     16384 x 7168, 1 x 128 blocks: an activation / gradient with its 128 x 1-blocked transpose (wgrad operand)
  w       7168 x 2048, 128 x 128 blocks: a weight and its transpose (dgrad operand)
  experts 32 x 2048 x 7168, 128 x 128 blocks: a batch of expert weights and their transposes
Arms:
  lib       one b200_fp8_quantize call (q, scales, qt and, for 1 x 128, the transposed scales), preallocated outputs
  lib_q     the same without the transposed output
  torch     the torch-ops route of the repo's tests and probes: x.float(), amax over each block, divide, cast, and
            for the transposed output .t().contiguous() and a second quantisation (1 x 128) or a transposed copy of q
            (128 x 128)
  copy      a device-to-device copy (torch.Tensor.copy_) of a uint8 buffer, moving the same bytes as `lib`
Bytes moved are counted from the shapes: x read once, q and qt written once, and the scales.  Every arm is warmed up;
the arms alternate inside each round, each timed with CUDA events around a batch of calls; each figure is the median
over rounds with the spread (min, max).  Prints the card name, power limit and max SM clock, and writes everything as
JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs  # noqa: E402

SHAPES = {"act": ((16384, 7168), 1), "w": ((7168, 2048), 128), "experts": ((32, 2048, 7168), 128)}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except OSError:
        pass
    return torch.cuda.get_device_name(0) + " (power limit not readable)"


def torch_1x128(x):
    *lead, r, k = x.shape
    g = x.float().reshape(*lead, r, k // 128, 128)
    s = g.abs().amax(dim=-1) / 448
    return (g / s[..., None]).reshape(x.shape).to(torch.float8_e4m3fn), s


def torch_128x128(w):
    *lead, n, k = w.shape
    g = w.float().reshape(*lead, n // 128, 128, k // 128, 128)
    s = g.abs().amax(dim=(-3, -1)) / 448
    return (g / s[..., :, None, :, None]).reshape(w.shape).to(torch.float8_e4m3fn), s


def arms(gemm, x, block):
    lead, (m, k) = tuple(x.shape[:-2]), tuple(x.shape[-2:])
    G = lead[0] if lead else 1
    qm, qk = m // 128, k // 128
    q = torch.empty(x.shape, dtype=torch.float8_e4m3fn, device="cuda")
    qt = torch.empty(lead + (k, m), dtype=torch.float8_e4m3fn, device="cuda")
    s = torch.empty(lead + ((m if block == 1 else qm), qk), device="cuda")
    st = torch.empty(lead + (k, qm), device="cuda") if block == 1 else None
    e = (lambda t: t.stride(0) if lead else 0)
    stream = torch.cuda.current_stream().cuda_stream

    def lib(trans=True):
        t = (qt.data_ptr(), m, e(qt)) if trans else (None, 0, 0)
        ts = (st.data_ptr(), st.stride(-2), st.stride(-1), e(st)) if trans and st is not None else (None, 0, 0, 0)
        rc = gemm.lib.b200_fp8_quantize(1, 0, block, m, k, G, x.data_ptr(), k, e(x), q.data_ptr(), k, e(q), s.data_ptr(),
                                        s.stride(-2), s.stride(-1), e(s), *t, *ts, stream)
        assert rc == 0, rc

    def torch_ops():
        if block == 1:
            torch_1x128(x)
            torch_1x128(x.transpose(-2, -1).contiguous())
        else:
            wq, _ = torch_128x128(x)
            wq.transpose(-2, -1).contiguous()

    moved = x.numel() * x.element_size() + 2 * x.numel() + 4 * (s.numel() + (st.numel() if st is not None else 0))
    moved_q = x.numel() * x.element_size() + x.numel() + 4 * s.numel()
    src = torch.empty(moved // 2, dtype=torch.uint8, device="cuda")
    dst = torch.empty_like(src)
    return {"lib": (lib, moved), "lib_q": (lambda: lib(False), moved_q), "torch": (torch_ops, moved),
            "copy": (lambda: dst.copy_(src), 2 * (moved // 2))}


def timing(gemm, rounds, calls):
    out = {}
    for name, (shape, block) in SHAPES.items():
        torch.manual_seed(1)
        x = torch.randn(shape, device="cuda", dtype=torch.bfloat16)
        a = arms(gemm, x, block)
        for f, _ in a.values():                       # warm-up: modules, allocator, torch's kernels
            for _ in range(3):
                f()
        torch.cuda.synchronize()
        times = {k: [] for k in a}
        for _ in range(rounds):
            for k, (f, _) in a.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(calls):
                    f()
                e.record()
                torch.cuda.synchronize()
                times[k].append(s.elapsed_time(e) / calls)
        row = {"shape": list(shape), "block": f"{'1' if block == 1 else '128'}x128"}
        for k, (_, moved) in a.items():
            ms = statistics.median(times[k])
            row[k] = dict(ms=ms, spread_ms=[min(times[k]), max(times[k])], bytes=moved, gb_s=moved / ms / 1e6)
        row["lib_over_copy_bw"] = row["lib"]["gb_s"] / row["copy"]["gb_s"]
        row["torch_over_lib_time"] = row["torch"]["ms"] / row["lib"]["ms"]
        out[name] = row
        print(json.dumps({name: row}), flush=True)
        del a, x
        torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--calls", type=int, default=10)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    gemm = _libs.load_pkg()
    res = {"card": card(), "torch": torch.__version__}
    print(res["card"], flush=True)
    res["timing"] = timing(gemm, args.rounds, args.calls)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
