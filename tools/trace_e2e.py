"""Device timeline of the END-TO-END loop (StepDriver: H2D + graph replay + loss hand-off per step), from the
in-kernel %globaltimer tracer: per step, first-kernel start, last-kernel end and the idle gap to the next step."""
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
B = 300
spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
sess = TrainingSession(zoo.build("simple_dnn"), "x:0", "y:0", spec, acquire_lock=lock, engine="b200", seed=0, devices=[0]).open()
eng = sess.make_engine(torch.device("cuda", 0))
rng = np.random.default_rng(0)
rows = 50100
X = rng.random((rows, 784), dtype=np.float32)
Y = np.eye(10, dtype=np.float32)[rng.integers(0, 10, rows)]
eng.load_partition(X, Y)
nb = rows // B
eng.train_contiguous([(k % nb) * B for k in range(40)], B, pull=True)
eng.finish()
N = 40
with DeviceTrace(1 << 15) as tr:
    eng.train_contiguous([((40 + k) % nb) * B for k in range(N)], B, pull=True)
    eng.finish()
rec = [r for r in tr.records() if int(r["kid"]) < 100]
rec.sort(key=lambda r: int(r["t0"]))
# a step starts with the pull / cast kernels and ends with push: split on push records (kid 6)
steps, cur = [], None
for r in rec:
    t0, t2, kid = int(r["t0"]), int(r["t2"]), int(r["kid"])
    if cur is None:
        cur = dict(start=t0, end=t2, push_seen=False)
    elif cur["push_seen"] and kid != 6:
        steps.append(cur)
        cur = dict(start=t0, end=t2, push_seen=False)
    cur["end"] = max(cur["end"], t2)
    if kid == 6:
        cur["push_seen"] = True
if cur:
    steps.append(cur)
# per-kernel view of one step in the middle of the run (CTA records grouped by kernel id)
mid = steps[len(steps) // 2]
names = {1: "gemm", 2: "cast", 3: "softmax", 4: "mse", 5: "argmax", 6: "push/post", 7: "pull"}
per = {}
for r in rec:
    t0, t1, t2, kid = int(r["t0"]), int(r["t1"]), int(r["t2"]), int(r["kid"])
    if mid["start"] <= t0 <= mid["end"]:
        k = per.setdefault(kid, dict(first_start=t0, last_end=t2, ctas=0, cta_us=[]))
        k["first_start"] = min(k["first_start"], t0); k["last_end"] = max(k["last_end"], t2); k["ctas"] += 1
        k["cta_us"].append((t2 - t1) / 1e3)
kern = {names.get(k, str(k)): dict(start_us=(v["first_start"] - mid["start"]) / 1e3, end_us=(v["last_end"] - mid["start"]) / 1e3, cta_records=v["ctas"],
                                   cta_us_median=float(np.median(v["cta_us"])), cta_us_max=float(np.max(v["cta_us"]))) for k, v in per.items()}
dur = np.array([(s["end"] - s["start"]) / 1e3 for s in steps])
gap = np.array([(steps[i + 1]["start"] - steps[i]["end"]) / 1e3 for i in range(len(steps) - 1)])
period = np.array([(steps[i + 1]["start"] - steps[i]["start"]) / 1e3 for i in range(len(steps) - 1)])
out = dict(kernels_mid_step=kern, steps=len(steps), busy_us_median=float(np.median(dur)), gap_us_median=float(np.median(gap)), period_us_median=float(np.median(period)),
           busy_us=[round(float(v), 2) for v in dur[:16]], gap_us=[round(float(v), 2) for v in gap[:16]],
           host_us_per_step={n: v / eng._driver.steps() / 1e3 for n, v in
                             zip(("wait_slot", "h2d_enqueue", "event_handoff", "graph_launch", "record"), eng._driver.host_ns())})
# raw pinned H2D of one minibatch on the copy stream, for reference
xs = torch.empty(B, 784, device="cuda")
cs = torch.cuda.Stream()
ev = [torch.cuda.Event(enable_timing=True) for _ in range(21)]
with torch.cuda.stream(cs):
    for i in range(20):
        ev[i].record(cs)
        xs.copy_(eng.X[i * B:(i + 1) * B], non_blocking=True)
    ev[20].record(cs)
cs.synchronize()
out["h2d_us_each"] = [round(ev[i].elapsed_time(ev[i + 1]) * 1e3, 1) for i in range(20)]
import os
out["slots"] = eng.SLOTS
out["block"] = os.environ.get("SPARKFLOW_DRIVER_BLOCK", "0")
print(json.dumps(out))
json.dump(out, open("bench_out/trace_e2e%s.json" % ("_lock" if lock else ""), "w"))
sess.close()
