"""Launch the wgmma GEMM a few times for an `ncu --set full` capture (one GPU, short).

    ncu --set full --clock-control none --import-source on -k regex:sf_gemm_kernel -s 4 -c 2 -o bench_out/prof_gemm \
        python tools/profile_gemm.py 4096 4096 4096
"""
import sys

import torch

sys.path.insert(0, ".")
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up

M, N, K = (int(v) for v in sys.argv[1:4]) if len(sys.argv) >= 4 else (4096, 4096, 4096)
pair = 1 if "--pair" in sys.argv else 0
C = native.cuda_ext()
C.set_pdl(0)
a = torch.randn(M, round_up(K, 8), device="cuda").to(torch.bfloat16)
b = torch.randn(N, round_up(K, 8), device="cuda").to(torch.bfloat16)
out = torch.zeros(M, round_up(N, 8), dtype=torch.bfloat16, device="cuda")
bias = torch.randn(N, device="cuda")
g = C.Gemm(dict(a=native.ptr(a), b=native.ptr(b), M=M, N=N, K=K, lda=a.shape[1], ldb=b.shape[1], out_bf16=native.ptr(out),
                ld_bf16=out.shape[1], bias=native.ptr(bias), act=1, pair=pair))
st = native.current_stream()
for _ in range(8):
    g.launch(st)
torch.cuda.synchronize()
print("gemm", M, N, K, "bn", g.bn, "grid", g.grid)
