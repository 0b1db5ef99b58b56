"""Front-end timeline of the end-to-end loop from CUDA timing events (SPARKFLOW_DRV_PROBE=1): per step, when its H2D
finished (copy stream), when the compute stream passed the hand-off, and when the step graph finished."""
import json
import os
import sys

import numpy as np
import torch

os.environ["SPARKFLOW_DRV_PROBE"] = "1"
sys.path.insert(0, ".")
from sparkflow_b200.models import zoo
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.session import TrainingSession

B = 300
spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
sess = TrainingSession(zoo.build("simple_dnn"), "x:0", "y:0", spec, acquire_lock="--lock" in sys.argv, engine="b200", seed=0, devices=[0]).open()
eng = sess.make_engine(torch.device("cuda", 0))
rng = np.random.default_rng(0)
rows = 50100
eng.load_partition(rng.random((rows, 784), dtype=np.float32), np.eye(10, dtype=np.float32)[rng.integers(0, 10, rows)])
nb = rows // B
N = 240
eng.train_contiguous([(k % nb) * B for k in range(N)], B, pull=True)
eng.finish()
p = np.asarray(eng._driver.probe(), dtype=np.float64).reshape(-1, 4)
p = p[np.argsort(p[:, 0])][40:]
step, ready, start, end = p.T
gap = start[1:] - end[:-1]                 # compute stream idle between consecutive graphs (front-end view)
h2d_late = ready[1:] - end[:-1]            # > 0: the step's H2D finished after the previous graph did
dur = end - start
out = dict(slots=eng.SLOTS, steps=len(p),
           period_us=float(np.median(np.diff(end))), period_mean_us=float(np.mean(np.diff(end))),
           dur_us_median=float(np.median(dur)), dur_us_p90=float(np.percentile(dur, 90)), dur_us_max=float(dur.max()),
           gap_us_median=float(np.median(gap)), gap_us_p90=float(np.percentile(gap, 90)), gap_us_max=float(gap.max()),
           h2d_late_frac=float(np.mean(h2d_late > 0)), h2d_late_us_p90=float(np.percentile(h2d_late, 90)),
           first_rows=[[round(float(v), 1) for v in r] for r in np.c_[step, ready - start[0], start - start[0], end - start[0]][:20]])
print(json.dumps(out))
json.dump(out, open("bench_out/e2e_probe_%s.json" % eng.SLOTS, "w"))
sess.close()
