"""One-CTA GEMM at 128- and 64-row tiles on the dense GEMMs of the flagship step (simple_dnn 784-256-256-10, batch 300),
each with the epilogue variant the step runs.

    python tools/bench_rows64.py [--reps=5] [--launches=400]

Each shape's GEMM is captured `launches` times back to back into one CUDA graph, which is replayed `reps` times between
CUDA events; the operands stay L2-resident, as they are in the step.  Reported per launch (µs, median over the replays),
with programmatic dependent launch off (kernel to kernel) and on (as in the step: the next GEMM's prologue overlaps this
one's epilogue).  Prints one JSON line per shape and the card's name and power limit.  Writes nothing."""
import json
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, ".")
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import round_up

FWD, LOSS, DGRAD, WGRAD = 1, 2, 3, 4
arg = lambda k, d: next((a.split("=", 1)[1] for a in sys.argv if a.startswith(f"--{k}=")), d)
REPS = int(arg("reps", "5"))
LAUNCHES = int(arg("launches", "400"))
B = 300
# (name, variant, M, N, K)
SHAPES = [("fwd0", FWD, B, 256, 784), ("fwd1", FWD, B, 256, 256), ("fwd2+loss", LOSS, B, 10, 256), ("dgrad2", DGRAD, B, 256, 10),
          ("dgrad1", DGRAD, B, 256, 256), ("wgrad0", WGRAD, 784, 256, B), ("wgrad1", WGRAD, 256, 256, B), ("wgrad2", WGRAD, 256, 10, B)]


def card():
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["sm_max_mhz"] = float(out[0]), float(out[1])
    except Exception as exc:  # noqa: BLE001 - reported, not fatal
        info["power_limit_error"] = f"{type(exc).__name__}: {exc}"
    return info


def bf16(rows, cols, g, fn=None):
    x = torch.randn(rows, cols, device="cuda", generator=g) * 0.5
    out = torch.zeros(rows, round_up(cols, 8), dtype=torch.bfloat16, device="cuda")
    out[:, :cols] = (fn(x) if fn else x).to(torch.bfloat16)
    return out


def gemm_dict(kind, M, N, K, keep):
    """the GEMM as the step builds it: its operands, outputs and epilogue inputs (kept alive in `keep`)"""
    g = torch.Generator(device="cuda").manual_seed(M + N + K)
    if kind == WGRAD:
        a, b = bf16(K, M, g), bf16(K, N, g)
        out = torch.zeros(M, N, device="cuda")
        keep += [a, b, out]
        return dict(a=native.ptr(a), b=native.ptr(b), M=M, N=N, K=K, lda=a.shape[1], ldb=b.shape[1], mn_major=1, out_f32=native.ptr(out),
                    ld_f32=N)
    a, b = bf16(M, K, g), bf16(N, K, g)
    out = torch.zeros(M, round_up(N, 8), dtype=torch.bfloat16, device="cuda")
    keep += [a, b, out]
    d = dict(a=native.ptr(a), b=native.ptr(b), M=M, N=N, K=K, lda=a.shape[1], ldb=b.shape[1], out_bf16=native.ptr(out), ld_bf16=out.shape[1])
    if kind in (FWD, LOSS):
        bias = torch.randn(N, device="cuda", generator=g)
        keep.append(bias)
        d["bias"] = native.ptr(bias)
    if kind == FWD:
        d["act"] = 1
    if kind in (LOSS, DGRAD):
        colsum = torch.zeros(N, device="cuda")
        keep.append(colsum)
        d["colsum"] = native.ptr(colsum)
    if kind == LOSS:
        y = torch.eye(N, device="cuda")[torch.randint(0, N, (M,), device="cuda", generator=g)]
        loss = torch.zeros(1, device="cuda")
        keep += [y, loss]
        d.update(loss_mode=1, target=native.ptr(y), ld_target=N, loss=native.ptr(loss))
    if kind == DGRAD:
        aux = bf16(M, N, g, fn=torch.relu)
        keep.append(aux)
        d.update(aux=native.ptr(aux), ld_aux=aux.shape[1], aux_act=1)
    return d


def time_graph(gm):
    """µs per launch: `LAUNCHES` launches captured in one graph, the median of `REPS` replays"""
    st = torch.cuda.Stream()
    with torch.cuda.stream(st):
        for _ in range(3):
            gm.launch(native.current_stream())
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st):
        for _ in range(LAUNCHES):
            gm.launch(native.current_stream())
    graph.replay()
    torch.cuda.synchronize()
    times = []
    for _ in range(REPS):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        graph.replay()
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1) * 1000.0 / LAUNCHES)
    return statistics.median(times), times


def main():
    assert torch.cuda.is_available(), "needs a GPU"
    C = native.cuda_ext()
    print(json.dumps({"card": card(), "sms": torch.cuda.get_device_properties(0).multi_processor_count, "launches": LAUNCHES,
                      "reps": REPS}), flush=True)
    keep = []
    for name, kind, M, N, K in SHAPES:
        d = gemm_dict(kind, M, N, K, keep)
        row = dict(gemm=name, M=M, N=N, K=K)
        for bm in (128, 64):
            gm = C.Gemm(dict(d, bm=bm, pair=0))
            assert gm.epi == kind, (name, gm.epi)
            row[f"grid_{bm}"] = list(gm.grid)
            row["bn"] = gm.bn
            for pdl in (0, 1):
                C.set_pdl(pdl)
                us, all_us = time_graph(gm)
                row[f"us_bm{bm}_pdl{pdl}"] = round(us, 3)
                row[f"spread_bm{bm}_pdl{pdl}"] = round(max(all_us) - min(all_us), 3)
        C.set_pdl(1)
        row["auto_bm"] = C.Gemm(dict(d, pair=0)).bm
        for pdl in (0, 1):
            row[f"saved_us_pdl{pdl}"] = round(row[f"us_bm128_pdl{pdl}"] - row[f"us_bm64_pdl{pdl}"], 3)
        assert C.read_error_code() == 0
        print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
