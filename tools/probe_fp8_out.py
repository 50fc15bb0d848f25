"""FP8 outputs of the FP8 GEMMs: torch's scale_result rule, and the fused 1 x 128 quantisation of C against its
unfused form.

--rule: what torch._scaled_mm on CUDA does with an FP8 out_dtype and scale_result.  Integer e4m3 operands with unit
input scales make the fp32 product exact; the output is compared with fp8(acc / s) and fp8(acc * s) for s in {0.5, 4},
and a product past the format's range shows whether torch saturates, gives inf or gives NaN.  Also reports whether
torch accepts a bias, and rowwise scales, with an FP8 output.

Timing (without --rule), at the MLP shape 16384 x 14336 x 4096 (rowwise scales, promoted) and DeepSeek-V3's
4096 x 7168 x 2048 (1 x 128 / 128 x 128 blockwise scales), GELU epilogue where the arm has one:
  fused     scaled_mm_quant: FP8 C and its 1 x 128 scales from the GEMM's epilogue (bias + GELU)
  fused_noact   the same without bias and activation
  unfused   the bf16-output scaled_mm, then the same quantisation in torch ops (amax, divide, cast)
  bf16      the bf16-output scaled_mm alone
  static / torch_static   scaled_mm(out_dtype=e4m3) with tensorwise scales against torch._scaled_mm's FP8 output
Every arm is warmed up; the arms alternate inside each round, each timed with CUDA events around a batch of calls; each
figure is the median over rounds, with the spread (min, max).

Prints the card name, power limit and max SM clock and writes everything as JSON to the file named by --out."""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "tests"))
import _libs  # noqa: E402

F8 = {"e4m3": torch.float8_e4m3fn, "e5m2": torch.float8_e5m2}


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True)
        if q.returncode == 0 and q.stdout.strip():
            return q.stdout.strip().splitlines()[0]
    except OSError:
        pass
    return torch.cuda.get_device_name(0) + " (power limit not readable)"


def bits(t):
    return t.view(torch.uint8).cpu()


def torch_rule():
    """torch._scaled_mm's FP8-output behaviour on this device."""
    out = {}
    gen = torch.Generator().manual_seed(3)
    m, n, k = 32, 32, 64
    a = torch.randint(-4, 5, (m, k), generator=gen).float()
    b = torch.randint(-4, 5, (n, k), generator=gen).float()
    acc = a @ b.t()                                                     # exact: |acc| <= 1024
    A = a.to(torch.float8_e4m3fn).cuda()
    B = b.to(torch.float8_e4m3fn).cuda()
    one = torch.ones((), device="cuda")
    fmax = {"e4m3": 448.0, "e5m2": 57344.0}
    for name, dt in F8.items():
        r = {}
        for pair in ((torch.float8_e4m3fn, torch.float8_e4m3fn), (torch.float8_e4m3fn, torch.float8_e5m2),
                     (torch.float8_e5m2, torch.float8_e4m3fn)):
            Ap, Bp = a.to(pair[0]).cuda(), b.to(pair[1]).cuda()
            pn = f"{str(pair[0])[-6:]}x{str(pair[1])[-6:]}"
            for s in (0.5, 4.0, 3.0, 0.3):
                try:
                    c = torch._scaled_mm(Ap, Bp.t(), one, one, scale_result=torch.tensor(s, device="cuda"), out_dtype=dt)
                except Exception as e:                                  # noqa: BLE001 - recorded as the finding
                    r[f"{pn}_{s}"] = f"refused: {e}"[:120]
                    continue
                cb = bits(c)
                sat = lambda x: x.clamp(-fmax[name], fmax[name]).to(dt)        # noqa: E731
                r[f"{pn}_{s}"] = dict(divides=bool(torch.equal(cb, bits(sat(acc / s)))),
                                      multiplies=bool(torch.equal(cb, bits(sat(acc * s)))),
                                      times_reciprocal=bool(torch.equal(cb, bits(sat(acc * (1 / torch.tensor(s)))))),
                                      ignored=bool(torch.equal(cb, bits(sat(acc)))))
                cf = c.float().cpu()
                nz = acc != 0
                r[f"{pn}_{s}"]["median_out_over_acc"] = float((cf[nz] / acc[nz]).median())
                r[f"{pn}_{s}"]["first"] = [(float(x), float(y)) for x, y in zip(acc.flatten()[:6], cf.flatten()[:6])]
        # overflow: |acc| = 64 * v^2 grows past 448 / 57344
        for v in (16.0, 128.0):
            Ab = torch.full((32, 64), v).to(torch.float8_e4m3fn).cuda()
            for sign in (1, -1):
                Bb = torch.full((32, 64), sign * v).to(torch.float8_e5m2 if name == "e5m2" else torch.float8_e4m3fn).cuda()
                key = f"overflow_acc_{sign * 64 * v * v:g}"
                try:
                    c = torch._scaled_mm(Ab, Bb.t(), one, one, scale_result=one, out_dtype=dt)
                    r[key] = dict(value=str(c.float()[0, 0].item()), bits=int(bits(c)[0, 0]))
                except Exception as e:                                  # noqa: BLE001
                    r[key] = f"refused: {e}"[:200]
        try:
            torch._scaled_mm(A, B.t(), one, one, bias=torch.zeros(n, device="cuda", dtype=torch.bfloat16),
                             scale_result=one, out_dtype=dt)
            r["bias_bf16"] = "accepted"
        except Exception as e:                                          # noqa: BLE001
            r["bias_bf16"] = f"refused: {e}"[:200]
        try:
            torch._scaled_mm(A, B.t(), torch.ones((m, 1), device="cuda"), torch.ones((1, n), device="cuda"),
                             out_dtype=dt)
            r["rowwise"] = "accepted"
        except Exception as e:                                          # noqa: BLE001
            r["rowwise"] = f"refused: {e}"[:200]
        out[name] = r
    return out


def timing(rounds):
    g = _libs.load_pkg()
    gen = torch.Generator(device="cuda").manual_seed(1)
    rows = []
    for shape, blockwise in (("16384x14336x4096", False), ("4096x7168x2048", True)):
        m, n, k = (int(v) for v in shape.split("x"))
        q, nb = -(-k // 128), -(-n // 128)
        x = torch.randn((m, k), device="cuda", generator=gen)
        W = torch.randn((n, k), device="cuda", generator=gen)
        if blockwise:
            sx = x.view(m, q, 128).abs().amax(dim=2) / 448
            Wp = torch.nn.functional.pad(W, (0, 0, 0, nb * 128 - n)).view(nb, 128, q, 128)
            sw = Wp.abs().amax(dim=(1, 3)) / 448
            xq = (x.view(m, q, 128) / sx[:, :, None]).view(m, k).to(torch.float8_e4m3fn)
            wq = (Wp / sw[:, None, :, None]).view(nb * 128, k)[:n].to(torch.float8_e4m3fn)
            sa, sb = sx.t().contiguous().t(), sw.t()
            del Wp
        else:
            sa = x.abs().amax(dim=1, keepdim=True) / 448
            sw = W.abs().amax(dim=1, keepdim=True) / 448
            xq, wq = (x / sa).to(torch.float8_e4m3fn), (W / sw).to(torch.float8_e4m3fn)
            sb = sw.t().contiguous()
        del x, W
        bias = torch.randn(n, device="cuda", generator=gen).bfloat16()
        qn = -(-n // 128)
        h8 = torch.empty((m, n), dtype=torch.float8_e4m3fn, device="cuda")
        hs = torch.empty((m, qn), device="cuda")
        hb = torch.empty((m, n), dtype=torch.bfloat16, device="cuda")
        one = torch.ones((), device="cuda")

        def fused():
            g.scaled_mm_quant(xq, wq.t(), sa, sb, bias=bias, activation="gelu", out=h8, out_scale=hs)

        def bf16():
            g.scaled_mm(xq, wq.t(), sa, sb, out=hb)

        def unfused():
            bf16()
            hv = torch.nn.functional.gelu(hb.float() + bias.float())          # the epilogue the fused call has
            hp = torch.nn.functional.pad(hv, (0, qn * 128 - n)).view(m, qn, 128)
            d = hp.abs().amax(dim=2) / 448
            d = torch.where(d == 0, torch.ones_like(d), d)
            h8.copy_((hp / d[:, :, None]).view(m, qn * 128)[:, :n].to(torch.float8_e4m3fn))
            hs.copy_(d)

        def fused_noact():
            g.scaled_mm_quant(xq, wq.t(), sa, sb, out=h8, out_scale=hs)

        arms = {"fused": fused, "fused_noact": fused_noact, "unfused": unfused, "bf16": bf16}
        if not blockwise:
            arms["static"] = lambda: g.scaled_mm(xq, wq.t(), one, one, out=h8)
            arms["torch_static"] = lambda: torch._scaled_mm(xq, wq.t(), one, one, scale_result=one,
                                                             out_dtype=torch.float8_e4m3fn)
        names = {}
        for a, f in arms.items():
            f(); f()
            names[a] = g.last_kernel() if a != "torch_static" else "cublasLt"
        torch.cuda.synchronize()
        iters = max(5, min(50, int(3e13 / (2.0 * m * n * k))))
        times = {a: [] for a in arms}
        for _ in range(rounds):
            for a, f in arms.items():
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(iters):
                    f()
                e.record()
                torch.cuda.synchronize()
                times[a].append(s.elapsed_time(e) / iters)
        row = dict(shape=shape, recipe="1x128-128x128" if blockwise else "rowwise promoted", iters=iters, names=names)
        for a in arms:
            row[a] = dict(ms=statistics.median(times[a]), spread_ms=[min(times[a]), max(times[a])])
        rows.append(row)
        print(shape, row["recipe"], " | ".join(f"{a} {row[a]['ms']:.3f} ms [{row[a]['spread_ms'][0]:.3f}, "
                                               f"{row[a]['spread_ms'][1]:.3f}]" for a in arms), flush=True)
        del xq, wq, h8, hs, hb
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rule", action="store_true", help="only measure torch's scale_result rule")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    info = card()
    cmd = " ".join(["python"] + sys.argv)
    print("card:", info, flush=True)
    print("command:", cmd, flush=True)
    print("torch:", torch.__version__, "cuda", torch.version.cuda, flush=True)
    res = dict(card=info, command=cmd, torch=torch.__version__, rule=torch_rule())
    print(json.dumps(res["rule"], indent=1), flush=True)
    if not args.rule:
        res["rounds"] = args.rounds
        res["timing"] = timing(args.rounds)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
