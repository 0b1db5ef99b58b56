"""Timeline of the flagship step from in-kernel %globaltimer stamps (device tracer, no profiler).

    python tools/trace_step.py [--lock] [--resident] [--model=simple_dnn] [--steps=4] [--out=DIR]

``--lock --resident`` traces what ``bench.py`` times for ``value``: lock mode, the HBM-resident partition and the native
StepDriver loop (back-to-back graph launches plus whatever the driver stages on the copy stream).  Without
``--resident`` the pinned-staging plan is replayed on its own."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from sparkflow_b200.models import zoo
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.session import TrainingSession
from sparkflow_b200.parallel.worker import B200Engine
from sparkflow_b200.utils.trace import DeviceTrace

BATCH = 300
lock = "--lock" in sys.argv
resident = "--resident" in sys.argv
arg = lambda k, d: next((a.split("=", 1)[1] for a in sys.argv if a.startswith(f"--{k}=")), d)
model = arg("model", "simple_dnn")
n_steps = int(arg("steps", "4"))
out_dir = arg("out", "bench_out")
spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
sess = TrainingSession(zoo.build(model), "x:0", "y:0" if model != "autoencoder" else None, spec, acquire_lock=lock, engine="b200",
                       seed=0, devices=[0]).open()
eng = sess.make_engine(torch.device("cuda", 0))
w = eng.w
st = w.stream
if resident:
    rng = np.random.default_rng(0)
    rows = 20 * BATCH
    D = w.plan.input_dim
    x = rng.random((rows, D), dtype=np.float32)
    if w.plan.target_is_input:
        y = None
    elif w.plan.loss == "sparse_softmax_xent":                    # one class index per row
        y = rng.integers(0, w.plan.layers[-1].out_features, (rows, 1)).astype(np.float32)
    else:
        y = np.eye(w.plan.label_dim, dtype=np.float32)[rng.integers(0, w.plan.label_dim, rows)]
    eng_r = B200Engine(w)
    eng_r.partition_mode = "resident"
    eng_r.load_partition(x, y)
    starts = [(k % 20) * BATCH for k in range(n_steps)]
    eng_r.train_contiguous(starts * 3, BATCH, pull=True)           # capture + warm up every slot
    eng_r.finish()
    plan, _ = w.build_plan(BATCH, 0, resident=(eng_r.Xd, eng_r.Yd))
    with torch.cuda.stream(st):
        with DeviceTrace(1 << 14) as tr:
            eng_r.train_contiguous(starts, BATCH, pull=True)
            st.synchronize()
            torch.cuda.synchronize()
else:
    plan, bufs = w.build_plan(BATCH, 0)
    bufs.x_stage.uniform_()
    if bufs.y_stage is not None:
        bufs.y_stage.zero_()
        bufs.y_stage[:, 3] = 1
    with torch.cuda.stream(st):
        for _ in range(6):
            w.run_plan(plan)
        st.synchronize()
        with DeviceTrace(1 << 14) as tr:
            for _ in range(n_steps):
                plan.replay(st.cuda_stream)
            st.synchronize()
rec = tr.records()
base = min(int(r["t0"]) for r in rec)
rows = []
for r in sorted(rec, key=lambda r: (int(r["t0"]))):
    rows.append(dict(kid=int(r["kid"]), block=int(r["block"]), t0=(int(r["t0"]) - base) / 1e3, t1=(int(r["t1"]) - base) / 1e3,
                     t2=(int(r["t2"]) - base) / 1e3))
# per-launch summary: CTAs of one launch leave griddepcontrol.wait together, so records of one kernel id are grouped by
# the proximity of their `ready` stamps (pre-launched successors START early and would otherwise be merged)
summ = []
by_kid = {}
for r in [x for x in rows if x["kid"] < 100]:
    by_kid.setdefault(r["kid"], []).append(r)
for kid, rs in by_kid.items():
    rs.sort(key=lambda r: r["t1"])
    cur = None
    for r in rs:
        if cur is None or r["t1"] > cur["last_ready"] + 0.3:
            cur = dict(kid=kid, start=r["t0"], ready=r["t1"], end=r["t2"], ctas=0, last_ready=r["t1"])
            summ.append(cur)
        cur["ctas"] += 1
        cur["start"] = min(cur["start"], r["t0"])
        cur["last_ready"] = r["t1"]
        cur["end"] = max(cur["end"], r["t2"])
summ.sort(key=lambda c: c["ready"])
names = {1: "gemm", 2: "cast", 3: "softmax", 4: "mse", 5: "argmax", 6: "push", 7: "pull", 8: "im2col", 9: "col2im", 10: "pool_fwd", 11: "pool_bwd", 12: "pool_gen_fwd", 13: "pool_gen_bwd",
         14: "act_bwd", 15: "sigmoid_xent", 16: "sparse_softmax_xent"}
print("card:", torch.cuda.get_device_name(0), "| plan:", plan.names())
print("%-8s %5s %9s %9s %9s %8s" % ("kernel", "ctas", "start_us", "ready_us", "end_us", "dur_us"))
for s in summ:
    print("%-8s %5d %9.2f %9.2f %9.2f %8.2f" % (names.get(s["kid"], s["kid"]), s["ctas"], s["start"], s["ready"], s["end"], s["end"] - s["ready"]))
pushes = [s["end"] for s in summ if s["kid"] == 6]
if len(pushes) > 1:
    print("step period (push end to push end, us):", ["%.2f" % (b - a) for a, b in zip(pushes, pushes[1:])])
PUSH_PHASES = (106, 107)
print("--- push phases, us from the push's ready: 106 = block 0 [grant seen, gradient loads returned, optimizer math done]; "
      "107 = last CTA [stores issued, done-counter arrival returned, tail done]")
for s in summ:
    if s["kid"] == 6:
        recs = [r for r in rows if r["kid"] in PUSH_PHASES and s["start"] <= r["t0"] <= s["end"]]
        print("push ready %9.2f, end %+6.2f: " % (s["ready"], s["end"] - s["ready"])
              + "  ".join("%d [%s]" % (r["kid"], ", ".join("%+6.2f" % (r[k] - s["ready"]) for k in ("t0", "t1", "t2"))) for r in recs))
print("--- gemm phases (block 0 of each gemm): 101 = MMA thread [role start, first operands, last MMA issued]; 102 = epilogue [wait start, acc ready, done]; 103 = [chunk 0 in registers, alpha+bias, activation]; 104 = [dropout, loss head, act'(aux)]; 105 = [padding+colsum, fp32 out, bf16 out]")
for r in rows:
    if r["kid"] >= 100 and r["block"] == 0 and r["kid"] not in PUSH_PHASES:
        print(r)
os.makedirs(out_dir, exist_ok=True)
json.dump(dict(summary=summ, rows=rows, plan=list(plan.names())),
          open(os.path.join(out_dir, "trace_step_%s%s%s.json" % (model, "_lock" if lock else "", "_resident" if resident else "")), "w"))
sess.close()
