"""Step time of any zoo model in the native engine and in the PyTorch interpreter engine.

    python tools/bench_zoo.py --model cnn_same [--steps 200] [--warmup 20] [--mode lock|hogwild] [--engines b200,torch]

Both arms use the timing of ``bench.py``'s ``value`` arm: seeded synthetic partition, minibatch 300, Adam(1e-3), warm-up
steps first, then K steps back to back between one pair of CUDA events on the engine's stream, ended by a device
synchronise.  ``b200``: HBM-resident partition, native step loop (one CUDA graph per step).  ``torch``: the
``engine="torch"`` interpreter (``graph/executor.py`` on cuda:0, parameter server on the host), which is what graphs
outside the compiled plan run on; its partition is moved to the GPU first so that the step does not time a host copy of
the minibatch.  Prints one JSON line with ms/step and samples/s per engine, the speedup of the native engine over the
interpreter, and the card's name and power limit read in the same run.  Writes nothing.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

BATCH = 300


def _card(index: int) -> dict:
    import torch

    info = {"name": torch.cuda.get_device_name(index), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                             stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30).stdout.strip().split(",")
        info["power_limit_w"], info["sm_max_mhz"] = float(out[0]), float(out[1])
    except Exception as exc:  # pragma: no cover - reported, not fatal
        info["power_limit_error"] = f"{type(exc).__name__}: {exc}"
    return info


def _partition(model: str, rows: int):
    import numpy as np

    from sparkflow_b200.graph.ir import GraphIR
    from sparkflow_b200.models import zoo
    from sparkflow_b200.models.compiler import compile_graph

    graph = zoo.build(model)
    ir = GraphIR.from_metagraph(graph)
    ph = {n.name: n for n in ir.nodes.values() if n.op in ("Placeholder", "PlaceholderV2")}
    in_dim = int(ph["x"].attrs["shape"][1])
    n_classes = int(ph["y"].attrs["shape"][1]) if "y" in ph else 0
    rng = np.random.default_rng(100)
    x = rng.random((rows, in_dim), dtype=np.float32)
    y = np.eye(n_classes, dtype=np.float32)[rng.integers(0, n_classes, rows)] if n_classes else None
    lp = compile_graph(ir, "x:0", "y:0") if n_classes else None
    if lp is not None and lp.loss == "sparse_softmax_xent":
        # a [None, 1] column of class indices (a StringIndexer output)
        y = rng.integers(0, lp.layers[-1].out_features, (rows, 1)).astype(np.float32)
    return graph, x, y


def run(model: str, engine: str, n_steps: int, warmup: int, lock: bool, rows: int) -> dict:
    import torch

    from sparkflow_b200.ops.optimizers import OptimizerSpec
    from sparkflow_b200.parallel.session import TrainingSession
    from sparkflow_b200.parallel.worker import B200Engine

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    graph, x, y = _partition(model, rows)
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001, beta1=0.9, beta2=0.999))
    sess = TrainingSession(graph, "x:0", "y:0" if y is not None else None, spec, acquire_lock=lock, iters=1, mini_batch=BATCH,
                           mini_stochastic_iters=1, shuffle=True, engine=engine, seed=1234, devices=[0]).open()
    if sess.engine_kind != engine:
        raise RuntimeError(f"{model}: asked for engine {engine!r}, the session runs {sess.engine_kind!r}")
    n_batches = rows // BATCH
    try:
        if engine == "b200":
            eng = B200Engine(sess.make_engine(dev).w)
            eng.partition_mode = "resident"
            eng.load_partition(x, y)
            st = eng.w.stream

            def steps(n, start):
                eng.train_contiguous([((start + k) % n_batches) * BATCH for k in range(n)], BATCH, pull=True)
        else:
            eng = sess.make_engine(dev)
            eng.load_partition(x, y)
            eng.X = eng.X.to(dev)
            eng.Y = None if eng.Y is None else eng.Y.to(dev)
            st = torch.cuda.current_stream(dev)

            def steps(n, start):
                for k in range(n):
                    r = ((start + k) % n_batches) * BATCH
                    eng.train(slice(r, r + BATCH), pull=True)

        steps(warmup, 0)
        eng.finish()
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        steps(n_steps, warmup)
        e1.record(st)
        eng.finish()
        torch.cuda.synchronize(dev)
        ms = e0.elapsed_time(e1) / n_steps
        loss = eng.last_loss() if engine == "b200" else None
        return {"ms_per_step": ms, "samples_per_s": BATCH / (ms / 1e3), "last_loss": loss}
    finally:
        sess.close()


def main() -> int:
    from sparkflow_b200.models import zoo

    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="cnn_same", choices=sorted(zoo.MODELS))
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--mode", default="lock", choices=["lock", "hogwild"])
    ap.add_argument("--engines", default="b200,torch", help="comma-separated subset of b200,torch")
    ap.add_argument("--partition-rows", type=int, default=12_000)
    args = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        print(json.dumps({"model": args.model, "error": "no CUDA device: bench_zoo.py measures on the GPU"}))
        return 1
    rows = max(args.partition_rows, 2 * BATCH)
    res = {"model": args.model, "batch": BATCH, "steps": args.steps, "warmup": args.warmup, "mode": args.mode, "card": _card(0)}
    for engine in args.engines.split(","):
        res[engine] = run(args.model, engine, args.steps, max(args.warmup, 3), args.mode == "lock", rows)
    if "b200" in res and "torch" in res:
        res["speedup_vs_torch"] = res["torch"]["ms_per_step"] / res["b200"]["ms_per_step"]
    print(json.dumps(res))
    return 0


if __name__ == "__main__":
    sys.exit(main())
