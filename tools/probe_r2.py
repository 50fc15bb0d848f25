"""Round-2 probe (GPU box): fp32 headline candidates.  Times every fp32 mode at N (default 4096) with
rotating operand sets, the F16X2 pre-pass pieces on their own (pack_a / pack_b) and the GEMM alone
(packed_ab), sweeps the raster group and the accumulation chunk, and checks the error of each
variant against the fp64 oracle on a row subset."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import _libs

g = _libs.load_pkg()
o = _libs.load_oracle()
dev = torch.device("cuda", 0)
N = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
R = 3
gen = torch.Generator(device=dev).manual_seed(7)
sets = [(torch.rand((N, N), device=dev, generator=gen) * 2 - 1, torch.rand((N, N), device=dev, generator=gen) * 2 - 1,
         torch.empty((N, N), device=dev)) for _ in range(R)]
rows = torch.arange(0, N, 61, device=dev)[:32]
truth = _libs.ref_f64(o, sets[0][0][rows].cpu().numpy(), sets[0][1].cpu().numpy())


def timeit(fn, iters=20, warm=3):
    for i in range(warm):
        fn(i)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for i in range(iters):
        fn(i)
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / iters


def err(C):
    got = C[rows].cpu().numpy()
    return float(np.abs(got - truth).max() / np.abs(truth).max())


out = {"N": N}
flops = 2.0 * N ** 3
for md, name in ((5, "f16x2"), (2, "bf16x3"), (3, "bf16x2"), (1, "tf32"), (0, "strict")):
    def fn(i, md=md):
        A, B, Cm = sets[i % R]
        g.gemm_f32(A, B, out=Cm, mode=md)
    ms = timeit(fn, iters=10 if md == 0 else 20)
    g.gemm_f32(sets[0][0], sets[0][1], out=sets[0][2], mode=md)
    out[name] = {"ms": ms, "tflops": flops / ms / 1e9, "kernel": g.last_kernel(), "rel_err": err(sets[0][2])}
    print(name, out[name], flush=True)

# F16X2 pieces
A, B, Cm = sets[0]
ms_pa = timeit(lambda i: g.PackedA(sets[i % R][0], mode=5).close(), iters=10)
ms_pb = timeit(lambda i: g.PackedB(sets[i % R][1], mode=5).close(), iters=10)
pas = [g.PackedA(s[0], mode=5) for s in sets]
pbs = [g.PackedB(s[1], mode=5) for s in sets]
ms_g = timeit(lambda i: g.gemm_f32_packed_ab(pas[i % R], pbs[i % R], sets[i % R][2]))
g.gemm_f32_packed_ab(pas[0], pbs[0], Cm)
out["f16x2_pieces"] = {"pack_a_ms_incl_malloc": ms_pa, "pack_b_ms_incl_malloc": ms_pb, "gemm_only_ms": ms_g,
                        "gemm_only_tflops": flops / ms_g / 1e9, "rel_err_packed": err(Cm)}
print(out["f16x2_pieces"], flush=True)

# raster group x chunk sweep on the GEMM alone
sweep = []
for grp in (2048, 4096):
    g.lib.b200_gemm_debug_set_group_rows(grp)
    for ck in (256, 512, 1024, 4096):
        g.lib.b200_gemm_debug_set_split_chunk(512, ck)
        ms = timeit(lambda i: g.gemm_f32_packed_ab(pas[i % R], pbs[i % R], sets[i % R][2]), iters=10)
        g.gemm_f32_packed_ab(pas[0], pbs[0], Cm)
        sweep.append({"group_rows": grp, "chunk_k": ck, "ms": ms, "tflops": flops / ms / 1e9, "rel_err": err(Cm)})
        print(sweep[-1], flush=True)
g.lib.b200_gemm_debug_set_group_rows(0)
g.lib.b200_gemm_debug_set_split_chunk(-1, -1)      # the built-in chunks of every split mode
out["f16x2_sweep"] = sweep
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(out, open(os.path.join(ROOT, "gpurun_out", f"probe_r2_{N}.json"), "w"), indent=1)

# ---- programmatic dependent launch on / off, and the 4-bit path ------------------------------------------
pdl = {}
bf = [((torch.rand(N, N, device=dev) - 0.5).bfloat16(), (torch.rand(N, N, device=dev) - 0.5).bfloat16()) for _ in range(R)]
i8 = [(torch.randint(-127, 128, (N, N), device=dev, dtype=torch.int8), torch.randint(-127, 128, (N, N), device=dev, dtype=torch.int8)) for _ in range(R)]
ob = [torch.empty(N, N, device=dev, dtype=torch.bfloat16) for _ in range(R)]
oi = [torch.empty(N, N, device=dev, dtype=torch.int32) for _ in range(R)]
for on in (1, 0, 1):
    g.lib.b200_gemm_debug_set_pdl(on)
    pdl[f"f16x2_step_ms_pdl{on}"] = timeit(lambda i: g.gemm_f32(sets[i % R][0], sets[i % R][1], out=sets[i % R][2], mode=5))
    pdl[f"bf16x3_step_ms_pdl{on}"] = timeit(lambda i: g.gemm_f32(sets[i % R][0], sets[i % R][1], out=sets[i % R][2], mode=2))
    pdl[f"bf16_obf16_ms_pdl{on}"] = timeit(lambda i: g.gemm_bf16(bf[i % R][0], bf[i % R][1], out=ob[i % R]))
    pdl[f"s8_ms_pdl{on}"] = timeit(lambda i: g.gemm_s8s32(i8[i % R][0], i8[i % R][1], out=oi[i % R]))
    print({k: round(v, 5) for k, v in pdl.items() if k.endswith(str(on))}, flush=True)
out["pdl"] = pdl
g.gemm_f32(sets[0][0], sets[0][1], out=sets[0][2], mode=5)
out["f16x2_rel_err_after_pdl"] = err(sets[0][2])
del bf, i8, ob, oi
mx = {}
for n in (4096, 8192):
    A = torch.rand(n, n, device=dev) * 2 - 1
    B = torch.rand(n, n, device=dev) * 2 - 1
    t_qa = timeit(lambda i: g.mxf4_quantize(A), iters=5)
    t_qb = timeit(lambda i: g.mxf4_quantize(B, transpose=True), iters=5)
    qa, sfa, _, _ = g.mxf4_quantize(A)
    qb, sfb, _, _ = g.mxf4_quantize(B, transpose=True)
    Cm = torch.empty(n, n, device=dev)
    t = timeit(lambda i: g.gemm_mxf4(qa, sfa, qb, sfb, n, n, n, out=Cm))
    mx[n] = {"gemm_ms": t, "tflops": 2.0 * n ** 3 / t / 1e9, "quantize_a_ms_incl_malloc": t_qa, "quantize_b_t_ms_incl_malloc": t_qb}
    print("mxf4", n, mx[n], flush=True)
    del A, B, qa, qb, sfa, sfb, Cm
out["mxf4"] = mx
json.dump(out, open(os.path.join(ROOT, "gpurun_out", f"probe_r2_{N}.json"), "w"), indent=1)
