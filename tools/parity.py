#!/usr/bin/env python
"""Convergence parity: the bf16 sm_90a engine vs the fp32 oracle, same init, same minibatch sequence.

The reference computes in fp32 (TF-1.x CPU kernels); the engine runs its GEMMs in bf16 with fp32 accumulation and
keeps fp32 master weights / optimizer state.  This tool trains the same model both ways on LEARNABLE synthetic data
(10 Gaussian blobs in 784-D for the classifiers, low-rank data for the autoencoders) for >= 500 steps, one optimizer step
per push, and records the two loss curves, the final losses / accuracies and the weight distance.

    python tools/parity.py --steps 600 --out bench_out/parity.json        (needs an H100)
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def blobs(n, d, c, rng, noise=1.0):
    # overlapping classes: the Bayes error is a few percent, so the loss stays well away from zero
    centers = rng.normal(0, 1, (c, d)).astype(np.float32) * 0.07
    lab = rng.integers(0, c, n)
    x = centers[lab] + noise * rng.normal(0, 1, (n, d)).astype(np.float32)
    return x.astype(np.float32), np.eye(c, dtype=np.float32)[lab], lab


def lowrank(n, d, r, rng):
    z = rng.random((n, r)).astype(np.float32)
    a = rng.random((r, d)).astype(np.float32) / r
    return np.clip(z @ a, 0, 1).astype(np.float32)


def run(model: str, steps: int, batch: int, lr: float, lock: bool):
    import torch

    from sparkflow_b200.graph.executor import GraphProgram
    from sparkflow_b200.graph.ir import GraphIR
    from sparkflow_b200.models import zoo
    from sparkflow_b200.ops.optimizers import OptimizerSpec
    from sparkflow_b200.parallel.param_server import LocalTransport, ParameterServer
    from sparkflow_b200.parallel.session import TrainingSession
    from sparkflow_b200.parallel.worker import TorchEngine

    rng = np.random.default_rng(42)
    classifier = model in ("simple_dnn", "cnn")
    n = 6000
    if classifier:
        X, Y, lab = blobs(n, 784, 10, rng)
        tf_label = "y:0"
    else:
        X, Y, lab, tf_label = lowrank(n, 784, 12, rng), None, None, None
    graph = zoo.build(model)
    ir = GraphIR.from_metagraph(graph)
    w0 = GraphProgram(ir).init_weights(seed=7)
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=lr))
    # ---- bf16 engine ----
    sess = TrainingSession(graph, "x:0", tf_label, spec, acquire_lock=lock, engine="b200", seed=7, initial_weights=w0, devices=[0]).open()
    eng = sess.make_engine(torch.device("cuda", 0))
    eng.load_partition(X, Y)
    # ---- fp32 oracle (PyTorch autograd interpreter of the same MetaGraph, fp32 everywhere, same Adam formula) ----
    ps = ParameterServer(w0, spec, acquire_lock=lock)
    ref = TorchEngine(ir, "x:0", tf_label, LocalTransport(ps), device="cuda")
    ref.load_partition(X, Y)
    nb = n // batch
    curve = []
    every = max(1, steps // 12)
    for k in range(steps):
        r0 = (k % nb) * batch
        rows = slice(r0, r0 + batch)
        eng.train(rows, pull=True)
        ref.train(rows, pull=True)
        if (k + 1) % every == 0 or k == 0:
            eng.finish()
            curve.append({"step": k + 1, "bf16_engine_loss": float(eng.partition_loss()), "fp32_oracle_loss": float(ref.partition_loss())})
    eng.finish()
    wg, wr = sess.weights(), ps.weights()
    rel = float(np.sqrt(sum(((a - b) ** 2).sum() for a, b in zip(wg, wr))) / np.sqrt(sum((b ** 2).sum() for b in wr)))
    out = {"model": model, "steps": steps, "batch": batch, "lr": lr, "lock": lock, "curve": curve, "weight_rel_l2_distance": rel}
    if classifier:
        prog = GraphProgram(ir)
        out["bf16_engine_accuracy"] = float((prog.forward("out:0", {"x:0": X}, wg).numpy() == lab).mean())
        out["fp32_oracle_accuracy"] = float((prog.forward("out:0", {"x:0": X}, wr).numpy() == lab).mean())
    sess.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=600)
    ap.add_argument("--batch", type=int, default=300)
    ap.add_argument("--models", default="simple_dnn,autoencoder,cnn")
    ap.add_argument("--out", default="bench_out/parity.json")
    args = ap.parse_args()
    res = []
    for m in args.models.split(","):
        res.append(run(m, args.steps, args.batch, 1e-3 if m != "cnn" else 1e-3, lock=True))
        print(json.dumps(res[-1]))
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    json.dump(res, open(args.out, "w"), indent=1)
    md = ["# bf16 engine vs fp32 oracle: loss curves on learnable synthetic data (same init, same minibatch order, Adam)", ""]
    for r in res:
        md += [f"## {r['model']} ({r['steps']} steps, batch {r['batch']}, lr {r['lr']}, lock mode)", "", "| step | bf16 engine loss | fp32 oracle loss | rel diff |", "|---|---|---|---|"]
        for c in r["curve"]:
            a, b = c["bf16_engine_loss"], c["fp32_oracle_loss"]
            md.append(f"| {c['step']} | {a:.5f} | {b:.5f} | {abs(a - b) / max(abs(b), 1e-9):.3%} |")
        md.append("")
        md.append(f"weights: relative L2 distance {r['weight_rel_l2_distance']:.4f}" +
                  (f"; accuracy bf16 {r['bf16_engine_accuracy']:.4f} vs fp32 {r['fp32_oracle_accuracy']:.4f}" if "bf16_engine_accuracy" in r else ""))
        md.append("")
    open(os.path.splitext(args.out)[0] + ".md", "w").write("\n".join(md))


if __name__ == "__main__":
    main()
