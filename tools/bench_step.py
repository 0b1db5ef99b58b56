"""Device-side microbenchmarks: wgmma GEMM vs torch.matmul, and the compiled training step."""
import json
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import compile_graph
from sparkflow_b200.ops import native
from sparkflow_b200.ops.layout import ParamLayout, round_up
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs


def time_fn(fn, iters=50, warm=5):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters * 1e3  # us


def bench_gemm(C, M, N, K, bn=0):
    a = torch.randn(M, round_up(K, 8), device="cuda").to(torch.bfloat16)
    b = torch.randn(N, round_up(K, 8), device="cuda").to(torch.bfloat16)
    out = torch.zeros(M, round_up(N, 8), dtype=torch.bfloat16, device="cuda")
    g = C.Gemm(dict(a=native.ptr(a), b=native.ptr(b), M=M, N=N, K=K, lda=a.shape[1], ldb=b.shape[1], bn=bn,
                    out_bf16=native.ptr(out), ld_bf16=out.shape[1]))
    st = native.current_stream()
    t_us = time_fn(lambda: g.launch(st))
    t_ref = time_fn(lambda: torch.matmul(a[:, :K], b[:, :K].t()))
    fl = 2.0 * M * N * K
    return dict(M=M, N=N, K=K, bn=g.bn, grid=list(g.grid), us=round(t_us, 2), tflops=round(fl / t_us / 1e6, 1),
                torch_us=round(t_ref, 2), torch_tflops=round(fl / t_ref / 1e6, 1))


def bench_step(name, tf_in, tf_lab, B, lock, pull_mode, steps=200):
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    ir = GraphIR.from_metagraph(zoo.build(name))
    lp = compile_graph(ir, tf_in, tf_lab)
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    dev = torch.device("cuda:0")
    master = MasterState(lay, spec, dev)
    master.load_weights(GraphProgram(ir).init_weights(seed=1))
    w = DeviceWorker(ir, tf_in, tf_lab, spec, master, acquire_lock=lock, pull_mode=pull_mode)
    plan, bufs = w.build_plan(B, 0)
    bufs.x_stage.uniform_()
    if bufs.y_stage is not None:
        bufs.y_stage.zero_()
        bufs.y_stage[:, 0] = 1
    st = w.stream
    with torch.cuda.stream(st):
        w.run_plan(plan)
        w.run_plan(plan)
        for _ in range(10):
            plan.replay(st.cuda_stream)
        st.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        plan.replay_n(st.cuda_stream, steps)
        e1.record(st)
        st.synchronize()
        us_graph = e0.elapsed_time(e1) / steps * 1e3
        e0.record(st)
        for _ in range(50):
            plan.run(st.cuda_stream)
        e1.record(st)
        st.synchronize()
        us_eager = e0.elapsed_time(e1) / 50 * 1e3
    res = dict(model=name, B=B, lock=lock, pull_mode=pull_mode, launches=len(plan), names=plan.names(),
               us_per_step_graph=round(us_graph, 2), us_per_step_eager=round(us_eager, 2),
               samples_per_s=round(B / us_graph * 1e6), params=ir.num_params(), counters=master.counters())
    master.close()
    return res


if __name__ == "__main__":
    C = native.cuda_ext()
    out = {"gemm": [], "step": []}
    if "--step-only" in sys.argv:
        tag = sys.argv[sys.argv.index("--tag") + 1] if "--tag" in sys.argv else "step"
        lock = "--lock" in sys.argv
        r = bench_step("simple_dnn", "x:0", "y:0", 300, lock, "copy", steps=300)
        r["tag"] = tag
        print(json.dumps(r), flush=True)
        sys.exit(0)
    for shp in [(300, 256, 784), (300, 256, 256), (300, 10, 256), (784, 256, 300), (256, 256, 300), (4096, 4096, 4096),
                (8192, 8192, 8192), (4096, 1000, 4096), (1024, 4096, 4096)]:
        out["gemm"].append(bench_gemm(C, *shp))
        print(json.dumps(out["gemm"][-1]), flush=True)
    for cfg in [("simple_dnn", "x:0", "y:0", 300, False, "copy"), ("simple_dnn", "x:0", "y:0", 300, True, "copy"),
                ("simple_dnn", "x:0", "y:0", 300, False, "direct"), ("autoencoder", "x:0", None, 256, False, "copy"),
                ("simple_dnn", "x:0", "y:0", 4096, False, "copy")]:
        out["step"].append(bench_step(*cfg))
        print(json.dumps(out["step"][-1]), flush=True)
    import os
    os.makedirs("bench_out", exist_ok=True)
    json.dump(out, open("bench_out/bench_step.json", "w"), indent=1)
