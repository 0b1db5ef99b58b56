"""Locked pull elision: a worker-applied push in lock mode also publishes into the pushing worker's replica, and the
worker's next pull copies nothing while no other push came in between.  Which path a pull took is read off a probe: one
replica element is overwritten before the pull, which only the copy restores."""
import numpy as np
import pytest
import torch

from push_helpers import wait_pushes
from sparkflow_b200.ops import native
from sparkflow_b200.ops.optimizers import OptimizerSpec
from test_step_gradients import DEV, UPDATE_TOL, _data, _model, _weights, _worker, oracle

NAME, B = "simple_dnn", 300          # the benchmarked step


def _second_worker(master, **kw):
    from sparkflow_b200.parallel.device_engine import DeviceWorker

    ir, _, label = _model(NAME)
    return DeviceWorker(ir, "x:0", label, master.spec, master, acquire_lock=True, shared=False, use_graphs=True, **kw)


def _engine(worker, X, Y):
    from sparkflow_b200.parallel.worker import B200Engine

    worker.use_graphs = True
    eng = B200Engine(worker)
    eng.load_partition(X, Y)
    return eng


def _bits0(worker):
    return worker.replica[:1].view(torch.int16)[0].item()


def _poison(worker):
    """overwrite replica element 0 with a value the publish never holds; returns its bits"""
    torch.cuda.synchronize()
    worker.replica[0] = -123.0
    torch.cuda.synchronize()
    return _bits0(worker)


def _pull(worker):
    """the worker's pull kernel with the arguments of its step plans; True when it copied (the probe was overwritten)"""
    bits = _poison(worker)
    worker.C.pull(worker._pull_args(), native.ptr(worker.sync_pull), 0, native.current_stream())
    torch.cuda.synchronize()
    assert worker.C.read_error_code() == 0
    copied = _bits0(worker) != bits
    if not copied:
        worker.replica[0] = worker.master.shadow[0]          # the copy was skipped: put the element back
        torch.cuda.synchronize()
    return copied


def _assert_replica_current(tag, master, worker):
    lay = master.layout
    torch.cuda.synchronize()
    assert torch.equal(worker.replica, master.shadow), f"{tag}: replica differs from the master's publish buffer"
    tail = master.state[lay.vec_offset:lay.vec_offset + lay.vec_count, 0]
    assert torch.equal(worker.vec_local[:lay.vec_count], tail), f"{tag}: fp32 tail differs from the master's parameters"
    assert int(master.ctrl[0]) == 0, f"{tag}: lock word {int(master.ctrl[0])}"


@pytest.mark.gpu
def test_own_push_makes_next_pull_skip_the_copy():
    """One worker, lock mode, five production steps: after each, the replica is the master's publish bit for bit and a
    pull copies nothing; the update of the five steps still tracks the float64 oracle's gradients."""
    from sparkflow_b200.parallel.param_server import LocalTransport, ParameterServer

    _, lp, _ = _model(NAME)
    spec = OptimizerSpec.from_tf_kwargs("gradient_descent", dict(learning_rate=0.05))
    w0 = _weights(NAME)
    X, Y = _data(NAME, 2 * B + 7, seed=B + 1)
    master, worker = _worker(NAME, w0, spec, lock=True)
    try:
        assert worker.own_publish
        eng = _engine(worker, X, Y)
        ref = LocalTransport(ParameterServer(w0, spec))
        assert _pull(worker), "the first pull must copy: the replica holds no version yet"
        steps = [slice(0, B), slice(B, 2 * B), np.random.default_rng(B).permutation(2 * B + 7)[:B], slice(7, B + 7), slice(0, B)]
        for k, rows in enumerate(steps):
            w_k = master.weights()
            eng.train(rows, pull=True)
            eng.finish()
            ref.push(oracle(lp, w_k, X[rows], Y[rows], emulate_bf16=True)[1])
            tag = f"step {k}"
            _assert_replica_current(tag, master, worker)
            assert int(worker.replica_version[0]) == int(master.ctrl[1]) == k + 1, tag
            assert not _pull(worker), f"{tag}: the pull after the worker's own push copied"
            assert int(worker.seen_version[0]) == k + 1 and int(master.ctrl[0]) == 0, tag
        assert wait_pushes(master, len(steps)) == len(steps)
        for a, b, a0, v in zip(master.weights(), ref.pull(), w0, lp.var_order):
            du, dr = a - a0, b - a0
            err = np.linalg.norm(du - dr) / np.linalg.norm(dr)
            assert np.isfinite(du).all() and err <= UPDATE_TOL, f"{v}: update off by {err:.2e}"
    finally:
        master.close()


@pytest.mark.gpu
def test_pull_after_another_workers_push_copies():
    """Two workers on one master, pushes interleaved: a pull after the other worker's push (or after its own dropped
    push) copies and leaves the replica equal to the publish at that moment; a pull right after its own push does not."""
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.01))
    w0 = _weights(NAME)
    X, Y = _data(NAME, 2 * B, seed=7)
    master, a = _worker(NAME, w0, spec, lock=True)
    try:
        b = _second_worker(master)
        ea, eb = _engine(a, X, Y), _engine(b, X, Y)
        for k in range(3):
            ea.train(slice(0, B), pull=True)
            ea.finish()
            assert not _pull(a), f"round {k}: the pull after a's own push copied"
            _assert_replica_current(f"round {k}, a after its push", master, a)
            eb.train(slice(B, 2 * B), pull=True)
            eb.finish()
            assert _pull(a), f"round {k}: the pull after b's push skipped the copy"
            _assert_replica_current(f"round {k}, a after b's push", master, a)
            assert not _pull(b), f"round {k}: the pull after b's own push copied"
        assert master.counters()["pushes"] == 6

        # a dropped push writes neither the replica nor its version: the pull after it copies
        ea.train(slice(0, B), pull=True)
        ea.finish()
        eb.train(slice(B, 2 * B), pull=True)
        eb.finish()
        mine = int(a.replica_version[0])
        bits = _poison(a)
        loss_out = torch.zeros(2, device=DEV)
        a.C.push(a._push_args(loss_out, drop=1), native.ptr(a.sync_push), 0, native.current_stream())
        torch.cuda.synchronize()
        c = master.counters()
        assert c["dropped"] == 1 and c["pushes"] == 8 and c["lock"] == 0, c
        assert int(a.replica_version[0]) == mine and _bits0(a) == bits
        assert _pull(a), "the pull after a dropped push skipped the copy"
        _assert_replica_current("after a dropped push", master, a)
    finally:
        master.close()


@pytest.mark.gpu
def test_worker_reading_between_pulls_keeps_the_pulled_weights():
    """A worker whose replica is read without a pull first (several minibatches per pull, a partition loss) does not
    publish into it: after a step it still holds the weights that step pulled."""
    spec = OptimizerSpec.from_tf_kwargs("adam", dict(learning_rate=0.01))
    w0 = _weights(NAME)
    X, Y = _data(NAME, B, seed=3)
    master, _ = _worker(NAME, w0, spec, lock=True)
    try:
        w = _second_worker(master, reads_between_pulls=True)
        assert not w.own_publish
        pulled = master.shadow.clone()
        eng = _engine(w, X, Y)
        eng.train(slice(0, B), pull=True)
        eng.finish()
        torch.cuda.synchronize()
        assert not torch.equal(master.shadow, pulled)
        assert torch.equal(w.replica, pulled)
        assert _pull(w), "a worker that does not publish into its replica must copy"
        _assert_replica_current("after the pull", master, w)
    finally:
        master.close()
