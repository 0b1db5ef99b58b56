"""Structure of the staged training step: the minibatch operands are prepared before the step graph starts (prep plan on
the staging stream), the graph starts with the pull on the main branch, and the last weight gradient runs on the main
branch right before the push."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from sparkflow_b200.graph.executor import GraphProgram
from sparkflow_b200.graph.ir import GraphIR
from sparkflow_b200.models import zoo
from sparkflow_b200.models.compiler import compile_graph
from sparkflow_b200.ops.layout import ParamLayout
from sparkflow_b200.ops.optimizers import OptimizerSpec
from sparkflow_b200.parallel.device_engine import DeviceWorker, MasterState, plan_publish_needs


def _worker(name="simple_dnn", lock=True):
    ir = GraphIR.from_metagraph(zoo.build(name))
    lp = compile_graph(ir, "x:0", "y:0")
    need_w, need_wt = plan_publish_needs(lp)
    lay = ParamLayout.build(ir.param_shapes(), need_w, need_wt)
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.001))
    master = MasterState(lay, spec, torch.device("cuda:0"))
    master.load_weights(GraphProgram(ir).init_weights(seed=1))
    return master, DeviceWorker(ir, "x:0", "y:0", spec, master, acquire_lock=lock, shared=False)


def _branch(name):
    return int(name.split("@")[1]) if "@" in name else 0


@pytest.mark.parametrize("resident", [False, True])
def test_staged_simple_dnn_plan_starts_with_pull_and_ends_with_main_branch_wgrad(resident):
    master, worker = _worker()
    X = torch.rand(600, 784, device="cuda:0")
    Y = torch.eye(10, device="cuda:0")[torch.randint(0, 10, (600,), device="cuda:0")]
    plan, bufs = worker.build_plan(300, 0, staged=True, resident=(X, Y) if resident else None)
    names = plan.names()
    assert not any(n.startswith(("cast_transpose", "gather_rows")) for n in names), names
    assert names[:2] == ["pull", "fwd0"], names
    assert names[-2:] == ["wgrad0", "push"], names
    wgrads = [n for n in names if n.startswith("wgrad")]
    assert len(wgrads) == 3
    branches = [_branch(n) for n in wgrads]
    assert all(a != b for a, b in zip(branches, branches[1:])), wgrads
    assert all(b in (1, 2) for b in branches[:-1]), wgrads
    prep = bufs.prep.names()
    assert prep == (["cast_transpose", "gather_rows"] if resident else ["cast_transpose"]), prep
    assert (bufs.idx is not None) == resident
    master.close()


def test_no_branches_gives_a_linear_staged_plan(monkeypatch):
    monkeypatch.setenv("SPARKFLOW_NO_BRANCHES", "1")
    master, worker = _worker()
    plan, _ = worker.build_plan(300, 0, staged=True)
    names = plan.names()
    assert not any("@" in n for n in names), names
    assert names[0] == "pull" and names[-1] == "push", names
    master.close()


def test_staged_and_in_graph_cast_steps_compute_the_same_gradient():
    """One step without push on the same rows: the staged plan (prep plan + step graph) and the self-contained plan (cast
    inside the graph) leave the same gradient buffer."""
    master, worker = _worker(lock=False)
    worker.use_graphs = False
    rng = np.random.default_rng(4)
    X = torch.from_numpy(rng.random((300, 784), dtype=np.float32))
    Y = torch.from_numpy(np.eye(10, dtype=np.float32)[rng.integers(0, 10, 300)])
    grads = []
    for staged in (False, True):
        plan, bufs = worker.build_plan(300, 0, with_push=False, staged=staged)
        with torch.cuda.stream(worker.stream):
            worker.grads.zero_()
            bufs.x_stage.copy_(X)
            bufs.y_stage.copy_(Y)
            if staged:
                bufs.prep.run(worker.stream.cuda_stream)
            plan.run(worker.stream.cuda_stream)
        worker.stream.synchronize()
        grads.append(worker.grads.clone().cpu())
    assert torch.count_nonzero(grads[0]) > 0
    torch.testing.assert_close(grads[1], grads[0], rtol=1e-2, atol=1e-4)
    master.close()
