"""GEMM throughput: the one-CTA wgmma kernel, the persistent 2-CTA kernel and cuBLAS (torch.matmul) on the same shapes.
CUDA-event timing, warm-up, L2 flushed between timed launches by rotating through operand sets larger than L2."""
import json
import sys

import torch

sys.path.insert(0, ".")
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up

C = native.cuda_ext()
C.set_pdl(0)
shapes = [(8192, 8192, 8192), (4096, 4096, 4096), (16384, 4096, 4096), (4096, 4096, 784), (2048, 4096, 4096)]
if len(sys.argv) > 1:
    shapes = [tuple(int(v) for v in a.split("x")) for a in sys.argv[1:]]
st = native.current_stream()
res = []
for M, N, K in shapes:
    nset = max(2, int(300e6 // ((M + N) * K * 2)) + 1)          # operand sets rotate so no launch finds its inputs in L2
    nset = min(nset, 8)
    As = [torch.randn(M, round_up(K, 8), device="cuda").to(torch.bfloat16) for _ in range(nset)]
    Bs = [torch.randn(N, round_up(K, 8), device="cuda").to(torch.bfloat16) for _ in range(nset)]
    out = torch.zeros(M, round_up(N, 8), dtype=torch.bfloat16, device="cuda")
    row = dict(M=M, N=N, K=K)
    flops = 2.0 * M * N * K

    def timed(fns, iters=20, warm=5):
        for i in range(warm):
            fns[i % len(fns)]()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            fns[i % len(fns)]()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters

    for name, pair in (("one_cta", 0), ("pair", 1)):
        try:
            gs = [C.Gemm(dict(a=native.ptr(a), b=native.ptr(b), M=M, N=N, K=K, lda=a.shape[1], ldb=b.shape[1], out_bf16=native.ptr(out),
                              ld_bf16=out.shape[1], pair=pair)) for a, b in zip(As, Bs)]
            ms = timed([(lambda g=g: g.launch(st)) for g in gs])
            row[name + "_tflops"] = flops / ms / 1e9
            row[name + "_ms"] = ms
        except Exception as exc:  # noqa: BLE001
            row[name + "_error"] = str(exc)[:200]
    ms = timed([(lambda a=a, b=b: torch.matmul(a, b.t())) for a, b in zip(As, Bs)])
    row["cublas_tflops"] = flops / ms / 1e9
    row["cublas_ms"] = ms
    # numerics spot check of the pair kernel against cuBLAS on the last operand set
    gs[-1].launch(st)
    torch.cuda.synchronize()
    ref = torch.matmul(As[-1], Bs[-1].t()).float()
    row["pair_max_rel_err_vs_cublas"] = float(((out[:, :N].float() - ref).abs().max() / ref.abs().max()).item())
    row["device_error"] = int(C.read_error_code())
    print(json.dumps(row), flush=True)
    res.append(row)
    del As, Bs, out
    torch.cuda.empty_cache()
json.dump(res, open("bench_out/bench_gemm.json", "w"), indent=1)
