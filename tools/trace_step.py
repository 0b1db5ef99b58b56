"""Timeline of one CUDA-graph replay of the flagship step (device tracer, no profiler)."""
import json
import sys

import numpy as np
import torch

sys.path.insert(0, ".")
from sparkflow_b200.models import zoo
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.session import TrainingSession
from sparkflow_b200.utils.trace import DeviceTrace

lock = "--lock" in sys.argv
model = next((a.split("=", 1)[1] for a in sys.argv if a.startswith("--model=")), "simple_dnn")
spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
sess = TrainingSession(zoo.build(model), "x:0", "y:0", spec, acquire_lock=lock, engine="b200", seed=0, devices=[0]).open()
eng = sess.make_engine(torch.device("cuda", 0))
w = eng.w
plan, bufs = w.build_plan(300, 0)
bufs.x_stage.uniform_()
bufs.y_stage.zero_()
bufs.y_stage[:, 3] = 1
st = w.stream
with torch.cuda.stream(st):
    for _ in range(6):
        w.run_plan(plan)
    st.synchronize()
    with DeviceTrace(1 << 14) as tr:
        for _ in range(3):
            plan.replay(st.cuda_stream)
        st.synchronize()
rec = tr.records()
launch = [r for r in rec if r["kid"] < 100]
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
names = {1: "gemm", 2: "cast", 3: "softmax", 4: "mse", 5: "argmax", 6: "push", 7: "pull", 8: "im2col", 9: "col2im", 10: "pool_fwd", 11: "pool_bwd"}
print("plan:", plan.names())
print("%-8s %5s %9s %9s %9s %8s" % ("kernel", "ctas", "start_us", "ready_us", "end_us", "dur_us"))
for s in summ:
    print("%-8s %5d %9.2f %9.2f %9.2f %8.2f" % (names.get(s["kid"], s["kid"]), s["ctas"], s["start"], s["ready"], s["end"], s["end"] - s["ready"]))
print("--- gemm phases (block 0 of each gemm): 101 = MMA thread [role start, first operands, last MMA issued]; 102 = epilogue [wait start, acc ready, done]; 103 = [chunk 0 in registers, alpha+bias, activation]; 104 = [dropout, loss head, act'(aux)]; 105 = [padding+colsum, fp32 out, bf16 out]")
for r in rows:
    if r["kid"] >= 100 and r["block"] == 0:
        print(r)
json.dump(dict(summary=summ, rows=rows), open("bench_out/trace_step_%s%s.json" % (model, "_lock" if lock else ""), "w"))
sess.close()
