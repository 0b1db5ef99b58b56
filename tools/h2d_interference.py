"""How much does a concurrent host->device transfer slow the step graph down?  Replays the captured simple_dnn step
back to back while a side stream (a) idles, (b) runs copy-engine DMAs of one minibatch."""
import json
import sys
import time

import numpy as np
import torch

sys.path.insert(0, ".")
from sparkflow_b200.models import zoo
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.session import TrainingSession

B = 300
spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
sess = TrainingSession(zoo.build("simple_dnn"), "x:0", "y:0", spec, acquire_lock=False, engine="b200", seed=0, devices=[0]).open()
eng = sess.make_engine(torch.device("cuda", 0))
w = eng.w
plan, bufs = w.build_plan(B, 0)
bufs.x_stage.uniform_()
bufs.y_stage.zero_()
bufs.y_stage[:, 3] = 1
st = w.stream
with torch.cuda.stream(st):
    for _ in range(5):
        w.run_plan(plan)
st.synchronize()
host = torch.rand(64, B, 784).pin_memory()
dst = torch.empty(4, B, 784, device="cuda")
side = torch.cuda.Stream()
nbytes = B * 784 * 4
N = 300
out = {}


def measure(name, side_fn, n_side):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s0.record(side)
    for i in range(n_side):
        side_fn(i)
    s1.record(side)
    e0.record(st)
    plan.replay_n(st.cuda_stream, N)
    e1.record(st)
    torch.cuda.synchronize()
    out[name] = dict(step_us=e0.elapsed_time(e1) * 1e3 / N, side_us_each=(s0.elapsed_time(s1) * 1e3 / n_side) if n_side else None)


measure("alone", lambda i: None, 0)
# side work sized to span the whole replay loop (~300 x 60 us = 18 ms): 600 copies of 0.94 MB
def dma(i):
    with torch.cuda.stream(side):
        dst[i % 4].copy_(host[i % 64], non_blocking=True)
measure("dma_h2d", dma, 600)
# side transfers alone (no step running)
s0, s1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize()
s0.record(side)
for i in range(200):
    dma(i)
s1.record(side)
torch.cuda.synchronize()
out["dma_alone"] = dict(side_us_each=s0.elapsed_time(s1) * 1e3 / 200, GBs=nbytes / (s0.elapsed_time(s1) * 1e-3 / 200) / 1e9)
assert torch.equal(dst[(199) % 4].cpu(), host[199 % 64])
print(json.dumps(out, indent=1))
json.dump(out, open("bench_out/h2d_interference.json", "w"), indent=1)
sess.close()
